"""oracle/sddmm_bsr_ref.py -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

Exact fixtures for the BSR sampled dense-dense product C = alpha * (op(A) * op(B)) o spy(C) + beta * C (sddmm_bsr.cu), in the manner
of oracle/sddmm_ref.py and oracle/bell_ref.py.

Format (cuSPARSE/sddmm_bsr): C is m x n in square bs x bs blocks; `off` holds m / bs + 1 block offsets and `col` the block column of
each stored block, both with index base `base`; `val` holds bnnz blocks of bs * bs values, each row-major or column-major inside the
block (the `order` argument of cusparseCreateBsr).  op(A) is m x k and op(B) k x n, passed here as int64 arrays in that orientation.

A and B hold small integers, alpha and beta are powers of two (or 0 / +-1), C0 even integers.  `check_exact` asserts that every
partial sum stays below 2^24 (2^53 for fp64) and that every output is an integer the output type holds exactly (bell_ref.OUT_LIMIT).
Any correct kernel then returns `reference` bit for bit, whatever its summation order.
"""
from __future__ import annotations

import ctypes as C
import json
import os

import numpy as np

from oracle.bell_ref import OUT_LIMIT

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SAMPLE = os.path.join(ROOT, "tests", "golden", "sddmm_bsr_sample.json")
LIMIT = dict(OUT_LIMIT, f64=(1 << 53) - 1)
SCALARS = [(1.0, 0.0), (-1.0, 1.0), (2.0, 0.5), (-2.0, -2.0)]      # (alpha, beta); beta == 0 is run on a NaN-filled C


def sample() -> dict:
    """sddmm_bsr's inputs, its golden (row-major blocks) and the three alternative goldens its source gives in comments"""
    with open(SAMPLE) as f:
        return json.load(f)["sddmm_bsr"]


def params(lib=None) -> dict:
    if lib is None:
        from cudalibrarysamples_b200 import lib as _lib
        lib = _lib.shim()
    k, s, t, f = C.c_int32(), C.c_int32(), C.c_int32(), C.c_int32()
    lib.b200sddmm_bsr_params(C.byref(k), C.byref(s), C.byref(t), C.byref(f))
    return dict(k_slab=k.value, stages=s.value, max_tile=t.value, fma_threads=f.value)


# ------------------------------------------------------------------------------------------------ converters
def block_rows(off, base=0) -> np.ndarray:
    """block-row of every stored block"""
    off = np.asarray(off, np.int64) - base
    return np.repeat(np.arange(len(off) - 1), np.diff(off))


def to_dense(m, n, bs, off, col, val, base=0, order="row", dtype=np.int64) -> np.ndarray:
    """m x n dense matrix of a BSR one (blocks row- or column-major inside)"""
    out = np.zeros((m, n), dtype)
    blocks = np.asarray(val).reshape(-1, bs, bs)
    if order == "col":
        blocks = blocks.transpose(0, 2, 1)
    for e, (r, c) in enumerate(zip(block_rows(off, base), np.asarray(col, np.int64) - base)):
        out[r * bs:(r + 1) * bs, c * bs:(c + 1) * bs] = blocks[e]
    return out


def from_dense(dense, bs, off, col, base=0, order="row") -> np.ndarray:
    """the values of the stored blocks (off, col) of `dense`, in the given block order"""
    blocks = [dense[r * bs:(r + 1) * bs, c * bs:(c + 1) * bs] for r, c in zip(block_rows(off, base), np.asarray(col, np.int64) - base)]
    blocks = np.array(blocks).reshape(-1, bs, bs)
    return (blocks.transpose(0, 2, 1) if order == "col" else blocks).ravel()


def to_scipy(m, n, bs, off, col, val, base=0, order="row"):
    import scipy.sparse as sp
    blocks = np.asarray(val).reshape(-1, bs, bs)
    if order == "col":
        blocks = blocks.transpose(0, 2, 1)
    return sp.bsr_matrix((blocks, np.asarray(col) - base, np.asarray(off) - base), shape=(m, n))


# ------------------------------------------------------------------------------------------------ patterns and values
def pattern(nbr, nbc, counts, seed, base=0):
    """block offsets / ascending distinct block columns with counts[r % len(counts)] blocks in block-row r (0 = an empty block-row)"""
    rng = np.random.default_rng(seed)
    cols, off = [], [0]
    for r in range(nbr):
        c = min(counts[r % len(counts)], nbc)
        cols.append(np.sort(rng.choice(nbc, c, replace=False)))
        off.append(off[-1] + c)
    col = np.concatenate(cols) if cols else np.zeros(0, np.int64)
    return np.array(off, np.int64) + base, col.astype(np.int64) + base


def values(m, n, k, bnnz, bs, seed, lo=-1, hi=1):
    """int64 op(A) (m x k), op(B) (k x n) and C0 (bnnz * bs * bs, even) in [lo, hi]"""
    rng = np.random.default_rng(seed)
    a = rng.integers(lo, hi + 1, (m, k), dtype=np.int64)
    b = rng.integers(lo, hi + 1, (k, n), dtype=np.int64)
    c0 = 2 * rng.integers(-3, 4, bnnz * bs * bs, dtype=np.int64)
    return a, b, c0


# ------------------------------------------------------------------------------------------------ reference
def products(bs, off, col, a, b, base=0, order="row", absolute=False) -> np.ndarray:
    """int64 (op(A) @ op(B)) on the stored blocks, in C's value layout (absolute: |op(A)| @ |op(B)|)"""
    if absolute:
        a, b = np.abs(a), np.abs(b)
    rows, cols = block_rows(off, base), np.asarray(col, np.int64) - base
    out = np.zeros((len(cols), bs, bs), np.int64)
    for e, (r, c) in enumerate(zip(rows, cols)):
        out[e] = a[r * bs:(r + 1) * bs] @ b[:, c * bs:(c + 1) * bs]
    return (out.transpose(0, 2, 1) if order == "col" else out).ravel()


def reference(bs, off, col, a, b, c0, alpha, beta, base=0, order="row") -> np.ndarray:
    """alpha * (op(A) @ op(B)) o spy(C) + beta * C0, exact in fp64 (integers and powers of two); beta == 0 ignores C0"""
    out = alpha * products(bs, off, col, a, b, base, order).astype(np.float64)
    if beta != 0:
        out = out + beta * np.asarray(c0, np.float64)
    return out


def check_exact(bs, off, col, a, b, c0, alpha, beta, out_kind, base=0):
    """every partial sum below 2^24 (2^53 for "f64"), and every output an integer `out_kind` ("f16", "bf16", "f32", "f64") holds"""
    acc_limit = (1 << 53) if out_kind == "f64" else (1 << 24)
    s = products(bs, off, col, a, b, base, absolute=True)
    for x in (alpha, beta):
        assert x == 0 or np.log2(abs(x)) == np.round(np.log2(abs(x)))
    bound = np.abs(alpha) * s + (np.abs(beta) * np.abs(np.asarray(c0, np.float64)) if beta != 0 else 0)
    assert (s < acc_limit).all() and (bound < acc_limit).all()
    ref = reference(bs, off, col, a, b, c0, alpha, beta, base)
    assert (ref == np.round(ref)).all() and (np.abs(ref) <= LIMIT[out_kind]).all()


def scipy_reference(m, n, bs, off, col, a, b, base=0, order="row") -> np.ndarray:
    """(op(A) @ op(B)) o spy(C) through scipy.sparse.bsr_matrix, in C's value layout"""
    ones = np.ones(len(col) * bs * bs)
    mask = to_scipy(m, n, bs, off, col, ones, base, order)
    prod = mask.multiply(a.astype(np.float64) @ b.astype(np.float64)).tobsr(blocksize=(bs, bs))
    return from_dense(prod.toarray(), bs, off, col, base, order)
