"""oracle/spsm_ref.py -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

numpy restatement of cusparseSpSM in this build (b200spsm_csr_analysis / b200spsm_csr_solve in
cudalibrarysamples_b200/csrc/spsm_csr.cu): C = alpha op(T)^-1 op(B) for a block of nrhs right-hand sides.

Analysis builds SpSV's plan (oracle/spsv_ref.py) and a level order: level[i] = 1 + max(level[j]) over the rows j that row i
depends on (0 without dependencies); order lists the rows by (level, position in the solve direction).

The solve computes each C(i, j) in this order, every operation rounded in the value type (no fused multiply-add):
  with W = tile(nrhs, c_row_major) and G = 32 / W entry groups, group g sums the products val[t_vidx[m]] * C(t_col[m], j) of the
  row's plan entries m = b + g, b + g + G, ... in ascending order starting from +0; the groups are then added by the xor tree
  (offsets 16, 8, ..., W between lanes, i.e. group g with group g ^ (o / W)), and C(i, j) = (alpha * op(B)(i, j) - s) / d_i
  (no division for unit).  So a result's bits depend on the plan and W only.
"""
from __future__ import annotations

import numpy as np

from oracle import spsv_ref as SR

plan = SR.plan
ascending = SR.ascending


def levels(rows, p, lower=True, transpose=False):
    """(level[rows], order[rows], number of levels) of plan p, as b200spsm_csr_analysis computes them."""
    t_off, t_col = p["t_off"].astype(np.int64), p["t_col"].astype(np.int64)
    lev = np.zeros(rows, np.int64)
    seq = range(rows) if ascending(lower, transpose) else range(rows - 1, -1, -1)
    for i in seq:
        deps = t_col[t_off[i]:t_off[i + 1]]
        lev[i] = lev[deps].max() + 1 if deps.size else 0
    pos = np.arange(rows) if ascending(lower, transpose) else rows - 1 - np.arange(rows)      # position in the solve direction
    order = np.lexsort((pos, lev)).astype(np.int32)
    return lev, order, int(lev.max()) + 1 if rows else 0


def tile(nrhs, c_row_major):
    """b200spsm_csr_tile: right-hand sides per tile of the solve kernel."""
    cap = 32 if c_row_major else 8
    w = 1
    while w < cap and w < nrhs:
        w *= 2
    return w


def solve(rows, off, col, val, opB, alpha=1.0, base=0, lower=True, unit=False, transpose=False, w=1, diag=None):
    """C (rows x nrhs, the value type) = alpha op(T)^-1 opB in the kernel's exact order for tile width w.  opB: rows x nrhs.
    diag: rows values replacing the stored diagonal (cusparseSpSM_updateMatrix DIAGONAL)."""
    val = np.asarray(val)
    dt = val.dtype.type
    opB = np.asarray(opB, dt)
    nrhs = opB.shape[1]
    p = plan(rows, off, col, base, lower, unit, transpose)
    _, order, _ = levels(rows, p, lower, transpose)
    t_off, t_col, t_vidx = p["t_off"], p["t_col"], p["t_vidx"]
    g_n = 32 // w
    a = dt(alpha)
    C = np.zeros((rows, nrhs), dt)
    with np.errstate(all="ignore"):
        for i in order:
            b, e = t_off[i], t_off[i + 1]
            n = e - b
            q = -(-n // g_n)
            prod = np.zeros((q * g_n, nrhs), dt)
            prod[:n] = val[t_vidx[b:e]][:, None] * C[t_col[b:e]]
            prod = prod.reshape(q, g_n, nrhs)
            s = np.zeros((g_n, nrhs), dt)
            for k in range(q):
                s = s + prod[k]
            o = 16
            while o >= w:
                s = s + s[np.arange(g_n) ^ (o // w)]
                o //= 2
            r = a * opB[i] - s[0]
            if not unit:
                d = dt(diag[i]) if diag is not None else (val[p["diag_vidx"][i]] if p["diag_vidx"][i] >= 0 else dt(np.nan))
                r = r / d
            C[i] = r
    return C


# ------------------------------------------------------------------------------------------------ fixtures
# The reference's spsm_csr toy (spsm_csr_example.c): the 4x4 matrix of spsv_csr, LOWER NON_UNIT, two column-major right-hand sides.
TOY_SPSM = dict(rows=4, nrhs=2, off=SR.TOY_SPSV["off"], col=SR.TOY_SPSV["col"], val=SR.TOY_SPSV["val"],
                B=np.array([1, 8, 23, 52, 1, 8, 23, 52], np.float32), C_result=np.array([1, 2, 3, 4, 1, 2, 3, 4], np.float32))


def long_rows_pattern(rows=200, seed=0):
    """Rows of 3 to 100 random columns over both triangles, every diagonal, and a first and a last row of 150 entries, mirrored
    into a symmetric pattern (so columns are as long as rows): each triangle and its transpose has rows far longer than 32, so every tile width sums several entries per group and the summation order shows in
    the bits (the stencils, the chain and the diagonal have at most two dependencies per row, where every order agrees)."""
    rng = np.random.default_rng(seed)
    r, c = [np.arange(rows)], [np.arange(rows)]
    for i in range(rows):
        k = 150 if i in (0, rows - 1) else int(rng.integers(3, 101))
        r.append(np.full(k, i))
        c.append(rng.choice(rows, k, replace=False))
    r, c = np.concatenate(r), np.concatenate(c)
    return SR.coo_to_csr(rows, np.concatenate([r, c]), np.concatenate([c, r]))


def fixtures():
    """(name, rows, off, col): the toy, 5-point stencils, the bidiagonal chain, the diagonal-only matrix and long random rows."""
    out = [("toy", 4, TOY_SPSM["off"], TOY_SPSM["col"])]
    for name, (off, col) in (("stencil5_6", SR.stencil5_pattern(6)), ("stencil5_9", SR.stencil5_pattern(9)),
                             ("chain", SR.chain_pattern(200)), ("diagonal", SR.diagonal_pattern(37)),
                             ("long_rows", long_rows_pattern())):
        out.append((name, off.size - 1, off, col))
    return out


def values(rows, off, col, dtype, seed=0):
    """Diagonally dominant values (every row stores its diagonal): off-diagonals uniform in [-1, 1) over the row's stored count, so
    a row's off-diagonals sum to less than 1 in magnitude and unit triangles stay well conditioned; |d_i| = 1 + sum of |row i|."""
    rng = np.random.default_rng(seed)
    off = np.asarray(off, np.int64)
    col = np.asarray(col, np.int64)
    r = np.repeat(np.arange(rows), np.diff(off))
    v = rng.uniform(-1, 1, off[-1]) / np.diff(off)[r]
    d = col == r
    v[d] = 0
    v[d] = (1.0 + np.bincount(r, weights=np.abs(v), minlength=rows))[r[d]] * rng.choice([-1, 1], int(d.sum()))
    return v.astype(dtype)
