"""oracle/spmm_bsr_ref.py -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

Exact fixtures for the BSR x dense product C = alpha * A * op(B) + beta * C (spmm_bsr.cu), in the manner of oracle/sddmm_bsr_ref.py,
whose BSR converters and patterns it reuses.  A is m x k in square bs x bs blocks (`off`, `col` with index base `base`, `val` holding
each block row- or column-major); op(B) is k x n, passed here as an int64 array in that orientation.

A and B hold small integers, alpha and beta are powers of two (or 0 / +-1), C0 even integers.  `check_exact` asserts that every
partial sum stays below 2^24 (2^53 for fp64) and that every output is an integer the output type holds exactly; any correct kernel
then returns `reference` bit for bit, whatever its summation order.

`walk` restates the kernels' work split in numpy: which CTA writes which block-row, directly or through carry slots.
"""
from __future__ import annotations

import ctypes as C

import numpy as np

from oracle.sddmm_bsr_ref import LIMIT, block_rows, pattern, to_dense, to_scipy  # noqa: F401  (re-exported for the tests)


def params(lib=None) -> dict:
    if lib is None:
        from cudalibrarysamples_b200 import lib as _lib
        lib = _lib.shim()
    v = [C.c_int32() for _ in range(7)]
    lib.b200spmm_bsr_params(*[C.byref(x) for x in v])
    keys = ("k_slab", "slabs_per_stage", "stages", "max_rows_per_cta", "chunk_min", "chunk_factor", "target_ctas")
    return dict(zip(keys, (x.value for x in v)))


def values(m, k, n, bnnz, bs, seed, lo=-1, hi=1):
    """int64 block values (bnnz * bs * bs), op(B) (k x n) and C0 (m x n, even) in [lo, hi]"""
    rng = np.random.default_rng(seed)
    val = rng.integers(lo, hi + 1, bnnz * bs * bs, dtype=np.int64)
    b = rng.integers(lo, hi + 1, (k, n), dtype=np.int64)
    c0 = 2 * rng.integers(-3, 4, (m, n), dtype=np.int64)
    return val, b, c0


def products(m, k, bs, off, col, val, b, base=0, order="row", absolute=False) -> np.ndarray:
    """int64 A @ op(B) (m x n); absolute: |A| @ |op(B)|"""
    a = to_dense(m, k, bs, off, col, val, base, order)
    if absolute:
        a, b = np.abs(a), np.abs(b)
    # fp64 BLAS: exact while every partial sum of the small-integer fixtures stays below 2^53 (check_exact bounds them far lower)
    return (a.astype(np.float64) @ np.asarray(b, np.float64)).astype(np.int64)


def reference(m, k, bs, off, col, val, b, c0, alpha, beta, base=0, order="row") -> np.ndarray:
    """alpha * A @ op(B) + beta * C0 (m x n), exact in fp64 for the fixtures above; beta == 0 ignores C0"""
    out = alpha * products(m, k, bs, off, col, val, b, base, order).astype(np.float64)
    if beta != 0:
        out = out + beta * np.asarray(c0, np.float64)
    return out


def check_exact(m, k, bs, off, col, val, b, c0, alpha, beta, out_kind, base=0, order="row"):
    """every partial sum below 2^24 (2^53 for "f64"), and every output an integer `out_kind` ("f16", "bf16", "f32", "f64") holds"""
    acc_limit = (1 << 53) if out_kind == "f64" else (1 << 24)
    s = products(m, k, bs, off, col, val, b, base, order, absolute=True)
    for x in (alpha, beta):
        assert x == 0 or np.log2(abs(x)) == np.round(np.log2(abs(x)))
    bound = np.abs(alpha) * s + (np.abs(beta) * np.abs(np.asarray(c0, np.float64)) if beta != 0 else 0)
    assert (s < acc_limit).all() and (bound < acc_limit).all()
    ref = reference(m, k, bs, off, col, val, b, c0, alpha, beta, base, order)
    assert (ref == np.round(ref)).all() and (np.abs(ref) <= LIMIT[out_kind]).all()


# ------------------------------------------------------------------------------------------------ the work split
def chunk(brows, bnnz, P, bs, n, batch=1) -> int:
    """stored blocks per piece: max(chunk_min, min(ceil(chunk_factor * bnnz / brows), ceil(work / target_ctas))), work counting one
    CTA per stored block, 64 rows of a block and 128 columns"""
    avg2 = -(-P["chunk_factor"] * bnnz // brows) if brows > 0 else 0
    work = bnnz * batch * (-(-bs // 64)) * (-(-n // 128))
    return max(P["chunk_min"], min(avg2, -(-work // P["target_ctas"])))


def walk(off, bnnz, P, bs, n, split=True, base=0, batch=1):
    """The kernels' walk over the stored blocks of one matrix.  Returns (ch, writes): one entry per write of a C block-row or a carry
    slot, ("C", block-row, writer) or ("carry", slot, writer), where the writer is a main-kernel CTA ("cta", unit) or the fix-up
    CTA ("fixup", block-row), and the pieces ("piece", block-row, first block, end) that the CTAs multiply, in walk order."""
    off = np.asarray(off, np.int64) - base
    brows = len(off) - 1
    ch = chunk(brows, bnnz, P, bs, n, batch)
    writes, pieces = [], []

    def cuts_ge(x):
        if x >= bnnz:
            return bnnz
        r = int(np.searchsorted(off, x, side="right") - 1)
        rs, re = int(off[r]), int(off[r + 1])
        return min(rs + -(-(x - rs) // ch) * ch, re)

    def run(unit, S, E):
        e = S
        while e < E:
            r = int(np.searchsorted(off, e, side="right") - 1)
            rs, re = int(off[r]), int(off[r + 1])
            pe = min(rs + ((e - rs) // ch + 1) * ch, re)          # the piece [e, pe)
            pieces.append(("piece", r, e, pe))
            if not split or re - rs <= ch:
                if pe == re:
                    writes.append(("C", r, ("cta", unit)))
            else:
                writes.append(("carry", 2 * (e // ch) + (1 if e == rs else 0), ("cta", unit)))
            e = pe

    if split:
        nchunks = -(-bnnz // ch)
        for c in range(nchunks):
            run(c, cuts_ge(c * ch), cuts_ge(min((c + 1) * ch, bnnz)))
        for r in range(brows):
            cnt = int(off[r + 1] - off[r])
            if cnt == 0 or cnt > ch:
                writes.append(("C", r, ("fixup", r)))
    else:
        for r in range(brows):
            if off[r + 1] == off[r]:
                writes.append(("C", r, ("cta", r)))
            run(r, int(off[r]), int(off[r + 1]))
    return ch, writes, pieces


def fixup_slots(off, r, ch, base=0):
    """the carry slots the fix-up adds for block-row r, in order"""
    off = np.asarray(off, np.int64) - base
    rs, re = int(off[r]), int(off[r + 1])
    return [2 * ((rs + p * ch) // ch) + (1 if p == 0 else 0) for p in range(-(-(re - rs) // ch))]
