"""oracle/spmm_csr_t_ref.py -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

The transposed plan of spmm_csr_t.cu restated in numpy, and what it must equal.

* `plan`: the kernels' algorithm -- a stable LSD radix sort of the entry indices by column, RT_BITS bits per pass, as many passes as
  cols - 1 needs bits (at least one) -- then the column pointers from the sorted columns and each CSC entry's row.
* `plan_scipy`: the same three arrays from scipy.sparse.csr_matrix.tocsc() (the CSC form, ascending rows within a column).
* `layout`: the workspace formula of b200spmm_csr_t_layout.
* `transpose`: the explicit CSR of A^T (tOff, tRow, val[perm]) -- the matrix whose opA = N product b200spmm_csr_t must equal bit for bit.

The product itself is checked with oracle/exact.py (fp32 / fp64) and oracle/spmm_csr16_ref.py (fp16 / bf16).
"""
from __future__ import annotations

import numpy as np
import scipy.sparse as sp

RT_BITS = 8
RT_TILE = 2048          # entries per tile of the sort (RT_THREADS x RT_ITEMS in spmm_csr_t.cu)


def passes(cols: int) -> int:
    bits = max(int(cols) - 1, 0).bit_length()
    return max(1, -(-bits // RT_BITS))


def plan(off, col, cols: int, base: int = 0):
    """(tOff, tRow, perm) int64, base 0, by the kernels' radix passes"""
    off = np.asarray(off, np.int64) - base
    keys = np.asarray(col, np.int64) - base
    nnz = keys.size
    idx = np.arange(nnz, dtype=np.int64)
    for p in range(passes(cols)):
        digit = (keys >> (p * RT_BITS)) & ((1 << RT_BITS) - 1)
        o = np.argsort(digit, kind="stable")           # stable: equal digits keep their order from the previous pass
        keys, idx = keys[o], idx[o]
    t_off = np.searchsorted(keys, np.arange(cols + 1), side="left").astype(np.int64)
    rows = off.size - 1
    t_row = np.searchsorted(off[1:], idx, side="right").astype(np.int64) if rows else idx
    return t_off, t_row, idx


def plan_scipy(off, col, rows: int, cols: int, base: int = 0):
    """(tOff, tRow, perm) from scipy's tocsc(), perm read back through the values 1 .. nnz"""
    off = np.asarray(off, np.int64) - base
    col = np.asarray(col, np.int64) - base
    nnz = col.size
    A = sp.csr_matrix((np.arange(1, nnz + 1, dtype=np.float64), col, off), shape=(rows, cols))
    A.has_sorted_indices = True                      # keep the stored order: tocsc() must not re-sort or merge anything
    T = A.tocsc()
    return T.indptr.astype(np.int64), T.indices.astype(np.int64), T.data.astype(np.int64) - 1


def transpose(off, col, val, rows: int, cols: int, base: int = 0):
    """A^T as a cols x rows CSR matrix, base 0: (tOff, tRow, val[perm])"""
    t_off, t_row, perm = plan(off, col, cols, base)
    return t_off, t_row, np.asarray(val)[perm]


def _up(b: int) -> int:
    return (b + 255) // 256 * 256


def layout(dtype: int, rows: int, cols: int, n: int, nnz: int, product_ws: int) -> dict:
    """b200spmm_csr_t_layout's offsets; product_ws: the opA = N entry point's own workspace bytes"""
    e = _up(4 * nnz)
    ntiles = -(-nnz // RT_TILE)
    L = {"t_off": 0, "t_row": _up(4 * (cols + 1))}
    L["perm"] = L["t_row"] + e
    L["scratch"] = L["perm"] + e
    scratch = 4 * e + _up(4 * 256 * ntiles) + _up(4 * 256)
    L["t_val"] = L["scratch"] + scratch
    L["ws"] = L["t_val"] + _up(nnz * {0: 4, 1: 8}.get(dtype, 2))
    L["total"] = L["ws"] + _up(product_ws)
    return L
