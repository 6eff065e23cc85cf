"""oracle/sddmm_ref.py -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

Exact fixtures for the sampled dense-dense product C = alpha * (op(A) * op(B)) o spy(C) + beta * C (sddmm_csr.cu), in the manner of
oracle/exact.py: A and B hold nonzero small integers, alpha and beta are powers of two (or 0 / +-1), C0 holds even integers, so
every partial sum of every dot product is an integer the value type holds exactly and any correct kernel returns the int64
reference bit for bit, whatever its split of K between lanes.  The "wide" fp64 variant takes 12-13-bit values: its products need
24-26 bits and its dot products more than fp32 has, so an accumulator narrowed to fp32 shows.  `check_exact` asserts the
precondition entry by entry.

`chunk_walk` is a numpy model of how sddmm_csr_kernel maps warps, steps and lanes to entries (from the constants of
b200sddmm_params): the CPU tests check that it computes every non-zero exactly once, on the row the offsets give it.
"""
from __future__ import annotations

import ctypes as C
import json
import os

import numpy as np

from . import exact as X

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SAMPLES = os.path.join(ROOT, "tests", "golden", "sddmm_samples.json")
MANTISSA = {"f32": 24, "f64": 53, "wide": 53}
NP_T = {"f32": np.float32, "f64": np.float64, "wide": np.float64}
SCALARS = X.SCALARS          # (alpha, beta); beta == 0 is run on a NaN-filled C


def samples() -> dict:
    """The toy inputs and goldens of cuSPARSE/sddmm_csr and sddmm_csr_batched (row-major A and B, NON_TRANSPOSE, alpha 1, beta 0)."""
    with open(SAMPLES) as f:
        return json.load(f)


def params(lib=None) -> dict:
    if lib is None:
        from cudalibrarysamples_b200 import lib as _lib
        lib = _lib.shim()
    w, u, v, g = C.c_int32(), C.c_int32(), C.c_int32(), C.c_int32()
    lib.b200sddmm_params(C.byref(w), C.byref(u), C.byref(v), C.byref(g))
    return dict(warp_chunk=w.value, unroll=u.value, vec_bytes=v.value, max_group=g.value)


def group(k: int, v: int, max_group: int = 32) -> int:
    """lanes per entry: the smallest power of two G with G * v >= k, at most max_group"""
    g = 1
    while g < max_group and g * v < k:
        g *= 2
    return g


def k_edges(P: dict, itemsize: int) -> list:
    """K values around the vector width, around every lane-group width of both paths, and several passes of the widest group"""
    v = P["vec_bytes"] // itemsize
    ks = {0, 1, 2, v - 1, v, v + 1}
    g = 1
    while g <= P["max_group"]:
        for w in (1, v):
            ks.update((g * w - 1, g * w, g * w + 1))
        g *= 2
    top = P["max_group"] * v
    ks.update((3 * top, 3 * top + v, 3 * top + 1))
    return sorted(k for k in ks if k >= 0)


# ------------------------------------------------------------------------------------------------ values and reference
def values(kind, m, n, k, nnz, seed):
    """int64 op(A) (m x k), op(B) (k x n) and C0 (nnz, even integers)"""
    rng = np.random.default_rng(seed)
    (alo, ahi), (blo, bhi), (_, chi) = X._RANGES[kind]
    a = X.nonzero_ints(rng, m * k, alo, ahi).reshape(m, k)
    b = X.nonzero_ints(rng, k * n, blo, bhi).reshape(k, n)
    c0 = 2 * rng.integers(-chi + 1, chi, nnz, dtype=np.int64) if chi > 1 else np.zeros(nnz, np.int64)
    return a, b, c0


def rows_of(off, base=0):
    off = np.asarray(off, np.int64) - base
    return np.repeat(np.arange(off.size - 1), np.diff(off))


def dots(off, col, a, b, base=0, absolute=False):
    """int64 op(A)(i, :) . op(B)(:, j) for every stored (i, j)"""
    r = rows_of(off, base)
    c = np.asarray(col, np.int64) - base
    a = np.abs(a) if absolute else a
    b = np.abs(b) if absolute else b
    if a.shape[1] == 0:
        return np.zeros(r.size, np.int64)
    return np.einsum("ek,ek->e", a[r].astype(np.int64), b[:, c].T.astype(np.int64))


def reference(off, col, a, b, c0, alpha, beta, base=0):
    """alpha * dot + beta * c0, exact: dot and c0 are integers, alpha / beta powers of two (fp64 holds every value here)"""
    s = dots(off, col, a, b, base)
    out = alpha * s.astype(np.float64)
    if beta != 0:
        out = out + beta * np.asarray(c0, np.float64)
    return out


def check_exact(off, col, a, b, c0, alpha, beta, p, base=0):
    """every partial sum, the scaled sum and the result stay below 2^p: no rounding anywhere, in any order"""
    s = dots(off, col, a, b, base, absolute=True)
    assert (s < (1 << p)).all()
    tot = np.abs(alpha) * s + (np.abs(beta) * np.abs(np.asarray(c0, np.float64)) if beta != 0 else 0)
    assert (2 * tot < float(1 << p)).all()


def scipy_reference(off, col, a, b, base=0):
    """the same product through scipy: (A @ B) sampled by the pattern, as a dense-then-gather (small sizes only)"""
    import scipy.sparse as sp
    m, n = a.shape[0], b.shape[1]
    nnz = len(col)
    pat = sp.csr_matrix((np.ones(nnz), np.asarray(col) - base, np.asarray(off) - base), shape=(m, n))
    full = pat.multiply(a.astype(np.float64) @ b.astype(np.float64)).tocsr()
    full.sort_indices()
    return full


# ------------------------------------------------------------------------------------------------ the kernel's index walk
def chunk_walk(off, nnz, k, v, P, base=0):
    """(visits per entry, row each visit used) of sddmm_csr_kernel: warp w owns entries [w * chunk, (w + 1) * chunk), finds the row
    of its first entry by binary search, then steps 32 / G entries at a time, `unroll` steps per iteration, each lane group walking
    its row forward."""
    off = np.asarray(off, np.int64) - base
    rows = off.size - 1
    lg = group(k, v, P["max_group"]).bit_length() - 1
    G, E, U, W = 1 << lg, 32 >> lg, P["unroll"], P["warp_chunk"]
    visits = np.zeros(nnz, np.int64)
    used_row = np.full(nnz, -1, np.int64)
    for n0 in range(0, nnz, W):
        n1 = min(n0 + W, nnz)
        lo, hi = 0, rows
        while hi - lo > 1:
            mid = (lo + hi) >> 1
            if off[mid] <= n0:
                lo = mid
            else:
                hi = mid
        for slot in range(E):                       # the lanes of one group share the walk of their slot
            r, rend = lo, off[lo + 1]
            for e0 in range(n0, n1, E * U):
                for u in range(U):
                    e = e0 + u * E + slot
                    if e >= n1:
                        continue
                    while rend <= e and r + 1 < rows:
                        r += 1
                        rend = off[r + 1]
                    visits[e] += 1
                    used_row[e] = r
    return visits, used_row
