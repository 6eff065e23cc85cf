"""numpy / scipy restatement of sparse <-> dense conversion (dense_convert.cu, DESIGN.md 3.24), on raw value bits.

Values are handled as (count, width) uint8 arrays so every type, NaN payloads included, compares bit for bit.  The dense operand
is a flat byte buffer of ld-strided lines in row- or column-major order; only the rows x cols window is written.
"""
from __future__ import annotations

import json
import os

import numpy as np

ORDER_COL, ORDER_ROW = 1, 2
GOLDEN = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "dense_samples.json")


def samples() -> dict:
    """The arrays of the three reference samples (sparse2dense_csr, dense2sparse_csr, dense2sparse_blockedell) and their results."""
    with open(GOLDEN) as f:
        return json.load(f)


def nonzero(bits: np.ndarray, part: int) -> np.ndarray:
    """"v != 0" of (count, width) value bits as the closed dense -> sparse analysis counts it, per part of `part` bytes (the
    width, or half of it for a complex type): the magnitude bits of any part set, so denormals, Inf and NaN are non-zero and +-0
    are zero -- except a 16-bit part whose magnitude bits exceed 0x7C00: that analysis reads fp16 and bf16 bits alike as fp16,
    where those are NaN, so it counts them as zero (for bf16: every value from about 2.7e36 up, Inf and NaN)."""
    if bits.shape[0] == 0:
        return np.zeros(0, bool)
    b = bits.reshape(bits.shape[0], -1, part).copy()
    b[:, :, part - 1] &= 0x7F                          # little-endian: the sign is the top bit of the last byte
    nz = b.any(axis=2)
    if part == 2:
        nz &= (b[:, :, 0].astype(np.uint32) | b[:, :, 1].astype(np.uint32) << 8) <= 0x7C00
    return nz.any(axis=1)


def window(m: int, n: int, ld: int, order: int) -> np.ndarray:
    """flat element index of each (i, j) of the m x n window"""
    i, j = np.meshgrid(np.arange(m), np.arange(n), indexing="ij")
    return (i * ld + j) if order == ORDER_ROW else (i + j * ld)


def scatter(dense: np.ndarray, m: int, n: int, ld: int, order: int, r, c, vals: np.ndarray) -> np.ndarray:
    """dense (elements x width bytes) with its window zeroed, then vals[k] stored at (r[k], c[k]) in order: the last of equal
    positions wins; positions outside the matrix are skipped"""
    out = dense.copy()
    out[window(m, n, ld, order).ravel()] = 0
    r, c = np.asarray(r, np.int64), np.asarray(c, np.int64)
    ok = (r >= 0) & (r < m) & (c >= 0) & (c < n)
    pos = (r * ld + c) if order == ORDER_ROW else (r + c * ld)
    out[pos[ok]] = vals[ok]                            # numpy assigns in order: the last duplicate wins
    return out


def csr_to_dense(dense, m, n, ld, order, off, ind, vals, base=0, csc=False):
    off, ind = np.asarray(off, np.int64) - base, np.asarray(ind, np.int64) - base
    major = np.repeat(np.arange(len(off) - 1), np.diff(off))
    r, c = (ind, major) if csc else (major, ind)
    return scatter(dense, m, n, ld, order, r, c, vals)


def bell_to_dense(dense, m, n, ld, order, bs, colind, vals, base=0):
    """Blocked-ELL A (colind[(m / bs) x slots], vals[m x ell_cols] row-major bytes) into dense; -1 slots never read"""
    colind = np.asarray(colind, np.int64).reshape((m + bs - 1) // bs, -1) - base
    ell_cols = colind.shape[1] * bs
    r, c, src = [], [], []
    for br in range(colind.shape[0]):
        for k, bc in enumerate(colind[br]):
            if bc < 0 or bc * bs >= n:
                continue
            for rr in range(min(bs, m - br * bs)):
                i = br * bs + rr
                for cc in range(bs):
                    r.append(i); c.append(bc * bs + cc); src.append(i * ell_cols + k * bs + cc)
    return scatter(dense, m, n, ld, order, r, c, vals[np.asarray(src, np.int64)] if src else vals[:0])


def dense_to_csr(dense, m, n, ld, order, part, base=0, csc=False):
    """(offsets, indices, value bytes) of the non-zeros of the window, in row order (CSR) or column order (CSC)"""
    idx = window(m, n, ld, order)
    vals = dense[(idx.T if csc else idx).ravel()]
    nz = nonzero(vals, part).reshape((n, m) if csc else (m, n))
    counts = nz.sum(axis=1)
    off = np.concatenate([[0], np.cumsum(counts)]) + base
    ind = np.nonzero(nz)[1] + base
    return off.astype(np.int64), ind.astype(np.int64), vals[nz.ravel()]


def dense_to_bell(dense, m, n, ld, order, bs, colind, ell_vals, base=0):
    """ell_vals (m x ell_cols elements, bytes) with every slot filled from the dense block it names; -1 slots get zeros"""
    colind = np.asarray(colind, np.int64).reshape((m + bs - 1) // bs, -1) - base
    ell_cols = colind.shape[1] * bs
    out = ell_vals.copy()
    for i in range(m):
        for cc in range(ell_cols):
            bc = colind[i // bs, cc // bs]
            j = bc * bs + cc % bs
            if bc < 0 or bc * bs >= n or j >= n:
                out[i * ell_cols + cc] = 0
            else:
                out[i * ell_cols + cc] = dense[i * ld + j if order == ORDER_ROW else i + j * ld]
    return out
