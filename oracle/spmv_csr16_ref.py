"""oracle/spmv_csr16_ref.py -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

Fixtures for the half-precision CSR SpMV y = alpha * A * x + beta * y (spmv_csr16.cu): A rows x cols CSR (`off`, `col` with index base
`base`, fp16 / bf16 values), x of A's type, y of A's type or fp32, fp32 accumulation.

* `reference_int`: the int64 product for integer data.  Its precondition check asserts that every value the kernel forms is an
  integer its type holds exactly: sum_k |a_rk| |x_k| < 2^24 bounds every fp32 product, run sum, piece sum and carry, alpha / beta are
  powers of two, and y stays within +-2048 for an fp16 y, +-256 for a bf16 y and below 2^24 for an fp32 y.  Any correct kernel then
  returns the reference bit for bit, whatever its summation order.
* `accumulate_f32`: the kernel's summation restated in numpy fp32, for any data whose products stay normal in fp32.  A product of two
  16-bit values is exact in fp32; a run sum is 0 + its products in order, a piece sum 0 + its runs' sums in order (a run the piece
  covers in part: 0 + the piece's products in it), and a row total 0 + its pieces in ascending chunk order.  Every add is an fp32
  add rounded to nearest even, as on the device, so this gives the kernel's bits.
* `walk`: both walks' work split restated -- which warp computes which piece, which carry slots are written and read, and who
  writes each row of y.
"""
from __future__ import annotations

import ctypes as C

import numpy as np

from oracle.spmm_csr16_ref import pattern  # noqa: F401  (the same CSR pattern helper)

LIMIT = {"f16": 2048, "bf16": 256, "f32": (1 << 24) - 1}
ACC_LIMIT = 1 << 24


def params(lib=None) -> dict:
    if lib is None:
        from cudalibrarysamples_b200 import lib as _lib
        lib = _lib.shim()
    v = [C.c_int32() for _ in range(3)]
    lib.b200spmv_csr16_params(*[C.byref(x) for x in v])
    return dict(zip(("chunk", "run", "warps"), (x.value for x in v)))


def values(rows, cols, nnz, seed, lo=-1, hi=1):
    """int64 values of A (nnz), x (cols) and y0 (rows, even) in [lo, hi]"""
    rng = np.random.default_rng(seed)
    val = rng.integers(lo, hi + 1, nnz, dtype=np.int64)
    x = rng.integers(lo, hi + 1, cols, dtype=np.int64)
    y0 = 2 * rng.integers(-3, 4, rows, dtype=np.int64)
    return val, x, y0


def products(off, col, val, x, base=0, absolute=False) -> np.ndarray:
    """int64 A @ x (rows); absolute: |A| @ |x|"""
    off = np.asarray(off, np.int64) - base
    col = np.asarray(col, np.int64) - base
    val = np.asarray(val, np.int64)
    x = np.asarray(x, np.int64)
    if absolute:
        val, x = np.abs(val), np.abs(x)
    rows = np.repeat(np.arange(len(off) - 1), np.diff(off))
    out = np.zeros(len(off) - 1, np.int64)
    np.add.at(out, rows, val * x[col])
    return out


def reference_int(off, col, val, x, y0, alpha, beta, y_kind, base=0) -> np.ndarray:
    """alpha * A @ x + beta * y0 as float64 (exact), after checking that the kernel's fp32 arithmetic is exact on this data and that
    y's type (y_kind "f16", "bf16" or "f32") holds every output; beta == 0 ignores y0"""
    for v in (alpha, beta):
        assert v == 0 or np.log2(abs(v)) == np.round(np.log2(abs(v))), v
    s = products(off, col, val, x, base, absolute=True)
    assert (s < ACC_LIMIT).all(), "a partial sum or carry would leave fp32's exact integers"
    out = alpha * products(off, col, val, x, base).astype(np.float64)
    if beta != 0:
        out = out + beta * np.asarray(y0, np.float64)
    bound = abs(alpha) * s + (abs(beta) * np.abs(np.asarray(y0, np.float64)) if beta != 0 else 0)
    assert (bound < ACC_LIMIT).all()
    assert (out == np.round(out)).all() and (np.abs(out) <= LIMIT[y_kind]).all(), "an output y's type does not hold exactly"
    return out


def accumulate_f32(off, col, val, x, chunk, run, base=0) -> np.ndarray:
    """acc_r of every row as the kernel forms it, in fp32 (see the module doc).  val and x hold values of A's 16-bit type (as floats).
    Adding +0 never changes an fp32 sum that starts from +0, so the entries a run or piece does not cover enter as +0."""
    off = np.asarray(off, np.int64) - base
    col = np.asarray(col, np.int64) - base
    m, nnz = len(off) - 1, int(off[-1])
    assert chunk % run == 0
    p = np.asarray(val, np.float32) * np.asarray(x, np.float32)[col]          # exact: 16-bit x 16-bit fits fp32
    e = np.arange(nnz, dtype=np.int64)
    row = np.repeat(np.arange(m, dtype=np.int64), np.diff(off))
    # sub-runs: a row's entries inside one run (runs never cross chunks)
    key = row * (nnz // run + 1) + e // run
    sub_start = np.flatnonzero(np.r_[True, key[1:] != key[:-1]]) if nnz else np.zeros(0, np.int64)
    sub_id = np.cumsum(np.r_[False, key[1:] != key[:-1]]) if nnz else np.zeros(0, np.int64)
    G = np.zeros((len(sub_start), run), np.float32)
    G[sub_id, e % run] = p
    u = np.zeros(len(sub_start), np.float32)
    for k in range(run):
        u = u + G[:, k]
    # pieces: a row's sub-runs inside one chunk
    s_row, s_e = row[sub_start], sub_start
    pkey = s_row * (nnz // chunk + 1) + s_e // chunk
    piece_id = np.cumsum(np.r_[False, pkey[1:] != pkey[:-1]]) if len(pkey) else np.zeros(0, np.int64)
    npieces = int(piece_id[-1]) + 1 if len(pkey) else 0
    P = np.zeros((npieces, chunk // run), np.float32)
    P[piece_id, (s_e % chunk) // run] = u
    S = np.zeros(npieces, np.float32)
    for k in range(chunk // run):
        S = S + P[:, k]
    # row totals: 0 + the pieces in ascending chunk order
    p_row = s_row[np.flatnonzero(np.r_[True, pkey[1:] != pkey[:-1]])] if len(pkey) else np.zeros(0, np.int64)
    first = np.searchsorted(p_row, np.arange(m))
    count = np.bincount(p_row, minlength=m)
    acc = np.zeros(m, np.float32)
    for j in range(int(count.max()) if m and npieces else 0):
        r = np.flatnonzero(count > j)
        acc[r] = acc[r] + S[first[r] + j]
    return acc


def round_to(acc, y_kind):
    """fp32 values rounded once to y's type (nearest even), as float64"""
    if y_kind == "f32":
        return np.asarray(acc, np.float32).astype(np.float64)
    if y_kind == "f16":
        return np.asarray(acc, np.float32).astype(np.float16).astype(np.float64)
    import torch
    return torch.from_numpy(np.asarray(acc, np.float32)).to(torch.bfloat16).double().numpy()


# ------------------------------------------------------------------------------------------------ the work split
def slot(kind, c):
    """carry slot of chunk c: in[c] (the piece of the row entering the chunk) = 2c, out[c] (the row leaving it) = 2c + 1"""
    return 2 * c + (1 if kind == "out" else 0)


def walk(off, chunk, split=True, base=0):
    """Both walks over one matrix.  Returns (writes, reads, pieces):
    writes: ("y", row, writer) and ("carry", slot, writer), the writer a chunk warp ("chunk", c) or a fix-up thread ("fixup", c);
    reads:  ("carry", slot, row, fix-up chunk) in the fix-up's order;
    pieces: (row, first entry, end, whose) for every piece whose sum reaches y, in the order its row adds it."""
    off = np.asarray(off, np.int64) - base
    m, nnz = len(off) - 1, int(off[-1])
    nch = max(1, -(-nnz // chunk))
    split = split and nch > 1
    writes, reads, pieces = [], [], []
    for c in range(nch):
        cs, ce = c * chunk, (c + 1) * chunk
        last = c == nch - 1
        lo = int(np.searchsorted(off, cs, side="left"))          # the first row starting at or after cs
        r = lo - 1 if lo > 0 and off[lo] > cs else lo
        while r < m and (last or off[r] < ce):
            rs, re = int(off[r]), int(off[r + 1])
            who = ("chunk", c)
            if rs < cs:                                          # entering: its piece is the fix-up's (split) or its owner's
                if split:
                    pieces.append((r, cs, min(re, ce), who))
                    writes.append(("carry", slot("in", c), who))
            elif re > ce:                                        # leaving
                pieces.append((r, rs, ce, who))
                if split:
                    writes.append(("carry", slot("out", c), who))
                else:
                    for c2 in range(c + 1, -(-re // chunk)):
                        pieces.append((r, c2 * chunk, min(re, (c2 + 1) * chunk), who))
                    writes.append(("y", r, who))
            else:
                if re > rs:
                    pieces.append((r, rs, re, who))
                writes.append(("y", r, who))
            r += 1
    if split:
        for c in range(nch - 1):
            cs, ce = c * chunk, (c + 1) * chunk
            r = int(np.searchsorted(off, ce - 1, side="right") - 1)
            rs, re = int(off[r]), int(off[r + 1])
            if rs < cs or re <= ce:
                continue
            reads.append(("carry", slot("out", c), r, c))
            for c2 in range(c + 1, -(-re // chunk)):
                reads.append(("carry", slot("in", c2), r, c))
            writes.append(("y", r, ("fixup", c)))
    return writes, reads, pieces
