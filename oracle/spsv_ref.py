"""oracle/spsv_ref.py -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

numpy restatement of the solve plan that cusparseSpSV_analysis builds in this build (b200spsv_csr_analysis in
cudalibrarysamples_b200/csrc/spsv_csr.cu), a plain sequential triangular solve, and exact fixtures for it.

The plan of op(A) with fill mode `lower` / diag type `unit`:
  t_off[rows+1], t_col[], t_vidx[]  the selected triangle of op(A) without its diagonal, as CSR; t_col is the row of y an
                                    entry depends on, t_vidx its index in the caller's values (0-based).  Row order:
                                    stored order (no transpose), ascending row of A (transpose; stored order among
                                    duplicates).  Columns outside [0, rows) are ignored.
  diag_vidx[rows]                   index of the first stored diagonal of row i, -1 for unit or when none is stored
  missing                           rows without a stored diagonal (counted for unit = 0 only)
The closed library's analysis is not observable, so this restatement defines the plan; the GPU output must equal it
bit for bit.
"""
from __future__ import annotations

import numpy as np


def plan(rows, off, col, base=0, lower=True, unit=False, transpose=False):
    off = np.asarray(off, np.int64) - base
    col = np.asarray(col, np.int64) - base
    nnz = int(off[-1]) if rows else 0
    k = np.arange(nnz, dtype=np.int64)
    r = np.repeat(np.arange(rows, dtype=np.int64), np.diff(off)) if rows else np.zeros(0, np.int64)
    c = col[:nnz]
    inside = (c >= 0) & (c < rows)
    diag_vidx = np.full(rows, -1, np.int32)
    if not unit:
        d = np.flatnonzero(inside & (c == r))
        first = np.unique(r[d], return_index=True)
        diag_vidx[first[0]] = d[first[1]]
    sel = inside & ((c < r) if lower else (c > r))
    if not transpose:
        trow, tcol, tk = r[sel], c[sel], k[sel]                # already in (row, stored position) order
    else:
        order = np.lexsort((k[sel], c[sel]))                   # by column of A, then stored position (== row of A)
        trow, tcol, tk = c[sel][order], r[sel][order], k[sel][order]
    t_off = np.zeros(rows + 1, np.int64)
    t_off[1:] = np.cumsum(np.bincount(trow, minlength=rows)) if rows else []
    missing = 0 if unit else int(np.count_nonzero(diag_vidx < 0))
    return dict(t_off=t_off.astype(np.int32), t_col=tcol.astype(np.int32), t_vidx=tk.astype(np.int32),
                diag_vidx=diag_vidx, missing=missing)


def ascending(lower, transpose):
    """Solve order: ascending rows for an effective lower triangle (LOWER, or UPPER with TRANSPOSE)."""
    return bool(lower) != bool(transpose)


def check_plan(rows, off, col, base, lower, unit, transpose, p):
    """The plan's invariants: every selected entry appears once, every dependency precedes its row in solve order, and
    t_vidx points at the stored entry (row, column) the plan claims."""
    o = np.asarray(off, np.int64) - base
    cc = np.asarray(col, np.int64) - base
    r_of = np.repeat(np.arange(rows), np.diff(o)) if rows else np.zeros(0, np.int64)
    t_off, t_col, t_vidx = p["t_off"].astype(np.int64), p["t_col"].astype(np.int64), p["t_vidx"].astype(np.int64)
    assert t_off[0] == 0 and np.all(np.diff(t_off) >= 0) and t_off[-1] == t_col.size == t_vidx.size
    assert np.unique(t_vidx).size == t_vidx.size                                   # each entry once
    i = np.repeat(np.arange(rows), np.diff(t_off)) if rows else np.zeros(0, np.int64)
    a_row, a_col = (i, t_col) if not transpose else (t_col, i)                      # the entry as stored in A
    assert np.array_equal(r_of[t_vidx], a_row) and np.array_equal(cc[t_vidx], a_col)
    assert np.all(t_col < i) if ascending(lower, transpose) else np.all(t_col > i)  # dependencies solved earlier
    inside = (cc >= 0) & (cc < rows)
    want = np.count_nonzero(inside & ((cc < r_of) if lower else (cc > r_of)))
    assert t_vidx.size == want
    d = p["diag_vidx"]
    ok = d >= 0
    assert np.all(r_of[d[ok]] == np.flatnonzero(ok)) and np.all(cc[d[ok]] == np.flatnonzero(ok))
    if unit:
        assert not ok.any()


def solve(rows, off, col, val, x, alpha=1.0, base=0, lower=True, unit=False, transpose=False, dtype=None):
    """op(T) y = alpha x row by row in solve order, in the value type (or dtype), summing in plan order."""
    dtype = np.dtype(dtype or np.asarray(val).dtype).type
    p = plan(rows, off, col, base, lower, unit, transpose)
    val = np.asarray(val, dtype)
    x = np.asarray(x, dtype)
    y = np.zeros(rows, dtype)
    a = dtype(alpha)
    order = range(rows) if ascending(lower, transpose) else range(rows - 1, -1, -1)
    for i in order:
        b, e = p["t_off"][i], p["t_off"][i + 1]
        s = np.sum(val[p["t_vidx"][b:e]] * y[p["t_col"][b:e]], dtype=dtype) if e > b else dtype(0)
        r = a * x[i] - s
        if not unit:
            r = r / val[p["diag_vidx"][i]]
        y[i] = r
    return y


# ------------------------------------------------------------------------------------------------ matrices
def stencil5_pattern(n):
    """The 5-point pattern on an n x n grid (cg_example.c / bicgstab_example.c), both triangles and the diagonal, sorted."""
    idx = np.arange(n * n).reshape(n, n)
    rows, cols = [idx.ravel()], [idx.ravel()]
    for a, b in ((idx[1:, :], idx[:-1, :]), (idx[:-1, :], idx[1:, :]), (idx[:, 1:], idx[:, :-1]), (idx[:, :-1], idx[:, 1:])):
        rows.append(a.ravel())
        cols.append(b.ravel())
    return coo_to_csr(n * n, np.concatenate(rows), np.concatenate(cols))


def chain_pattern(n):
    """Tridiagonal, both triangles stored: either triangle is a bidiagonal chain of n dependency levels."""
    i = np.arange(n)
    return coo_to_csr(n, np.concatenate([i, i[1:], i[:-1]]), np.concatenate([i, i[:-1], i[1:]]))


def diagonal_pattern(n):
    i = np.arange(n)
    return coo_to_csr(n, i, i)


def coo_to_csr(n, r, c):
    key = np.unique(np.asarray(r, np.int64) * max(n, 1) + np.asarray(c, np.int64))
    rr, cc = key // max(n, 1), key % max(n, 1)
    off = np.zeros(n + 1, np.int64)
    off[1:] = np.cumsum(np.bincount(rr, minlength=n))
    return off.astype(np.int32), cc.astype(np.int32)


# The reference's spsv_csr toy (spsv_csr_example.c:45-54): the full 4x4 matrix of the SpMV samples, LOWER NON_UNIT.
TOY_SPSV = dict(rows=4, off=np.array([0, 3, 4, 7, 9], np.int32), col=np.array([0, 2, 3, 1, 0, 2, 3, 1, 3], np.int32),
                val=np.array([1, 2, 3, 4, 5, 6, 7, 8, 9], np.float32), x=np.array([1, 8, 23, 52], np.float32),
                y_result=np.array([1, 2, 3, 4], np.float32))


# ------------------------------------------------------------------------------------------------ exact fixtures
def exact_case(rows, off, col, base=0, lower=True, unit=False, transpose=False, kind="f64", seed=0, alpha=2.0):
    """Values, y* and x such that op(T) y* = alpha x holds exactly and the solve must return y* bit for bit.

    Off-diagonal entries of T are nonzero integers in [-3, 3], diagonals are +-1, 2 or 4 (the division is exact), y* holds
    small integers ("wide": magnitudes 2^25 .. 2^26, so row sums need more than 24 bits and an fp32 accumulator would show), alpha is
    a power of two.  Every partial sum of every row, in any order, is bounded by the row's sum of |terms|, which is
    asserted to fit the type's integer range.  Stored entries outside T, and the stored diagonal under unit, are NaN:
    the solve must not read them.  Returns (val, x, y_star, alpha) in the value type."""
    dtype = np.float32 if kind == "f32" else np.float64
    rng = np.random.default_rng(seed)
    p = plan(rows, off, col, base, lower, unit, transpose)
    nnz = int(np.asarray(off)[-1]) - base if rows else 0
    val = np.full(nnz, np.nan)
    tv = rng.integers(1, 4, p["t_vidx"].size) * rng.choice([-1, 1], p["t_vidx"].size)
    val[p["t_vidx"]] = tv
    d = np.ones(rows, np.int64)
    if not unit:
        d = rng.choice([-1, 1, 2, 4], rows)
        assert np.all(p["diag_vidx"] >= 0), "NON_UNIT exact fixture needs a stored diagonal in every row"
        val[p["diag_vidx"]] = d
    if kind == "wide":                                     # |y*| in [2^25, 2^26]: every row sum needs more than 24 bits
        ys = rng.integers(2 ** 25, 2 ** 26 + 1, rows).astype(np.int64) * rng.choice([-1, 1], rows)
    else:
        ys = rng.integers(-8, 9, rows).astype(np.int64)
    t_off, t_col = p["t_off"].astype(np.int64), p["t_col"].astype(np.int64)
    i = np.repeat(np.arange(rows), np.diff(t_off)) if rows else np.zeros(0, np.int64)
    terms = tv.astype(np.int64) * ys[t_col]
    rowsum = d * ys
    np.add.at(rowsum, i, terms)
    abs_sum = np.abs(d * ys)
    np.add.at(abs_sum, i, np.abs(terms))
    limit = 2 ** 24 if dtype == np.float32 else 2 ** 53
    assert np.all(abs_sum < limit), "a partial sum would not be exact"          # precondition, row by row
    if kind == "wide":
        assert rows == 0 or np.any(abs_sum > 2 ** 24), "wide fixture needs row sums beyond fp32"
    x = (rowsum.astype(np.float64) / alpha).astype(dtype)
    assert np.all(x.astype(np.float64) * alpha == rowsum), "x is not exact"
    return val.astype(dtype), x, ys.astype(dtype), alpha
