"""oracle/spmm_csr16_ref.py -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

Fixtures for the half-precision CSR x dense product C = alpha * A * op(B) + beta * C (spmm_csr16.cu): A m x k CSR (`off`, `col` with
index base `base`, fp16 / bf16 values), op(B) k x n of A's type, C of A's type or fp32, fp32 accumulation.

* `reference_int`: the int64 product for integer data.  Its precondition check, row by row, asserts that every value the kernel forms
  is an integer its type holds exactly: sum_k |a_ik| |b_kj| < 2^24 bounds every fp32 partial sum, piece sum and carry, and the
  output stays within +-2048 for an fp16 C, +-256 for a bf16 C and below 2^24 for an fp32 C.  Any correct kernel then returns the
  reference bit for bit, whatever its summation order.
* `reference_f64`: the fp64 product with one rounding to C's type, for data that is not integer.
* `walk`: the kernels' work split restated in numpy -- which CTA writes which row, which carry slots each long row uses, and which
  fix-up reads them.
"""
from __future__ import annotations

import ctypes as C

import numpy as np

LIMIT = {"f16": 2048, "bf16": 256, "f32": (1 << 24) - 1}
ACC_LIMIT = 1 << 24


def params(lib=None) -> dict:
    if lib is None:
        from cudalibrarysamples_b200 import lib as _lib
        lib = _lib.shim()
    v = [C.c_int32() for _ in range(5)]
    lib.b200spmm_csr16_params(*[C.byref(x) for x in v])
    keys = ("piece", "lane_entries", "tile_rows", "warps", "max_cols_per_lane")
    return dict(zip(keys, (x.value for x in v)))


def pattern(lengths, cols, seed, base=0):
    """CSR offsets and ascending column indices (int64, index base `base`) with the given row lengths (each <= cols)"""
    rng = np.random.default_rng(seed)
    lengths = np.asarray(lengths, np.int64)
    off = np.concatenate([[0], np.cumsum(lengths)])
    col = np.concatenate([np.sort(rng.choice(cols, int(n), replace=False)) for n in lengths] + [np.zeros(0, np.int64)])
    return off + base, col.astype(np.int64) + base


def values(m, k, n, nnz, seed, lo=-1, hi=1):
    """int64 values of A (nnz), op(B) (k x n) and C0 (m x n, even) in [lo, hi]"""
    rng = np.random.default_rng(seed)
    val = rng.integers(lo, hi + 1, nnz, dtype=np.int64)
    b = rng.integers(lo, hi + 1, (k, n), dtype=np.int64)
    c0 = 2 * rng.integers(-3, 4, (m, n), dtype=np.int64)
    return val, b, c0


def products(off, col, val, b, base=0, absolute=False) -> np.ndarray:
    """int64 A @ op(B) (m x n); absolute: |A| @ |op(B)|"""
    off = np.asarray(off, np.int64) - base
    col = np.asarray(col, np.int64) - base
    val = np.asarray(val, np.int64)
    b = np.asarray(b, np.int64)
    if absolute:
        val, b = np.abs(val), np.abs(b)
    m = len(off) - 1
    rows = np.repeat(np.arange(m), np.diff(off))
    out = np.zeros((m, b.shape[1]), np.int64)
    np.add.at(out, rows, val[:, None] * b[col])
    return out


def reference_int(off, col, val, b, c0, alpha, beta, c_kind, base=0) -> np.ndarray:
    """alpha * A @ op(B) + beta * C0 as float64 (exact), after checking row by row that the kernel's fp32 arithmetic is exact on this
    data and that C's type (c_kind "f16", "bf16" or "f32") holds every output; beta == 0 ignores C0"""
    for x in (alpha, beta):
        assert x == 0 or np.log2(abs(x)) == np.round(np.log2(abs(x))), x
    s = products(off, col, val, b, base, absolute=True)
    assert (s < ACC_LIMIT).all(), "a partial sum or carry would leave fp32's exact integers"
    out = alpha * products(off, col, val, b, base).astype(np.float64)
    if beta != 0:
        out = out + beta * np.asarray(c0, np.float64)
    bound = np.abs(alpha) * s + (np.abs(beta) * np.abs(np.asarray(c0, np.float64)) if beta != 0 else 0)
    assert (bound < ACC_LIMIT).all()
    assert (out == np.round(out)).all() and (np.abs(out) <= LIMIT[c_kind]).all(), "an output C's type does not hold exactly"
    return out


def reference_f64(off, col, val, b, c0, alpha, beta, c_dtype, base=0):
    """alpha * A @ op(B) + beta * C0 in fp64 from the (already rounded) 16-bit inputs, rounded once to C's torch dtype; returns
    (rounded torch tensor, fp64 numpy result, fp64 sum_k |a_ik| |b_kj|)"""
    import torch
    off = np.asarray(off, np.int64) - base
    col = np.asarray(col, np.int64) - base
    m = len(off) - 1
    val = np.asarray(val, np.float64)
    b = np.asarray(b, np.float64)
    rows = np.repeat(np.arange(m), np.diff(off))
    prod = np.zeros((m, b.shape[1]))
    mag = np.zeros_like(prod)
    np.add.at(prod, rows, val[:, None] * b[col])
    np.add.at(mag, rows, np.abs(val)[:, None] * np.abs(b[col]))
    out = alpha * prod + (beta * np.asarray(c0, np.float64) if beta != 0 else 0)
    return torch.from_numpy(out).to(c_dtype), out, mag


# ------------------------------------------------------------------------------------------------ the work split
def pieces_of(rs, re, P):
    """the pieces [ps, pe) of the row [rs, re): its start plus multiples of P"""
    return [(ps, min(ps + P, re)) for ps in range(rs, re, P)]


def slot(ps, rs, P):
    """carry slot of the piece starting at ps of a long row starting at rs: [0] of chunk ps / P for a later piece, [1] for the first"""
    return 2 * (ps // P) + (1 if ps == rs else 0)


def walk(off, P, split=True, tile_rows=32, warps=8, base=0):
    """The kernels' walk over one matrix.  Returns (writes, reads, pieces):
    writes: ("C", row, writer) and ("carry", slot, writer) in launch order, the writer a row-tile CTA ("tile", t), a chunk warp
            ("chunk", c) or a fix-up warp ("fixup", c);
    reads:  ("carry", slot, row, fix-up chunk) in the fix-up's order;
    pieces: (row, first entry, end, whose) for every piece multiplied."""
    off = np.asarray(off, np.int64) - base
    m = len(off) - 1
    nnz = int(off[-1])
    nchunks = -(-nnz // P)
    split = split and nnz > P
    writes, reads, pieces = [], [], []

    def row_of(x):
        return int(np.searchsorted(off, x, side="right") - 1)

    for t in range(-(-m // tile_rows)):
        for r in range(t * tile_rows, min((t + 1) * tile_rows, m)):
            rs, re = int(off[r]), int(off[r + 1])
            if split and re - rs > P:
                pieces.append((r, rs, rs + P, ("tile", t)))
                writes.append(("carry", slot(rs, rs, P), ("tile", t)))
            else:
                for ps, pe in pieces_of(rs, re, P):
                    pieces.append((r, ps, pe, ("tile", t)))
                writes.append(("C", r, ("tile", t)))
    if not split:
        return writes, reads, pieces
    for c in range(nchunks):                                  # chunk warps: the later piece that starts in chunk c
        x = c * P
        r = row_of(x)
        rs, re = int(off[r]), int(off[r + 1])
        if re - rs <= P:
            continue
        ps = rs + -(-(x - rs) // P) * P
        if ps == rs or ps >= re:
            continue
        pieces.append((r, ps, min(ps + P, re), ("chunk", c)))
        writes.append(("carry", slot(ps, rs, P), ("chunk", c)))
    for c in range(nchunks):                                  # fix-up warps: the long row that starts in chunk c
        r = row_of(min((c + 1) * P, nnz) - 1)
        rs, re = int(off[r]), int(off[r + 1])
        if rs < c * P or re - rs <= P:
            continue
        for ps, _ in pieces_of(rs, re, P):
            reads.append(("carry", slot(ps, rs, P), r, c))
        writes.append(("C", r, ("fixup", c)))
    return writes, reads, pieces
