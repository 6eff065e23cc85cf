"""oracle/convert_ref.py -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

The conversions of convert.cu restated in numpy, and the data of cuSPARSE/coosort/coosort_example.c.

* `csr2csc`: the CSC form by spmm_csr_t_ref.plan_scipy (scipy's tocsc(): rows ascending within a column, duplicates in CSR order),
  in the input's base, with the values moved by the permutation.
* `coosort`: np.lexsort (stable) by (row, col) or (col, row), and P composed with the sort: P_out[i] = P_in[sigma(i)].
* `coo2csr` / `csr2coo`: searchsorted / repeat.
* `workspace`: the byte formulas of b200csr2csc_workspace_bytes / b200coosort_workspace_bytes.
"""
from __future__ import annotations

import json
import os

import numpy as np

from oracle import spmm_csr_t_ref as T

GOLDEN = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "coosort_sample.json")


def sample() -> dict:
    """coosort_example.c's input and golden arrays (tests/golden/coosort_sample.json)"""
    with open(GOLDEN) as f:
        return json.load(f)


def csr2csc(off, col, val, rows: int, cols: int, base: int = 0):
    """(cscColPtr, cscRowInd, cscVal) in the input's base; val None: cscVal None"""
    ptr, ind, perm = T.plan_scipy(off, col, rows, cols, base)
    return ptr + base, ind + base, None if val is None else np.asarray(val)[perm]


def coosort(rows, cols, P=None, by_row: bool = True):
    """(rows, cols, P) sorted by (row, col) -- or (col, row) -- stably; P defaults to the identity"""
    rows, cols = np.asarray(rows, np.int64), np.asarray(cols, np.int64)
    P = np.arange(rows.size, dtype=np.int64) if P is None else np.asarray(P, np.int64)
    sigma = np.lexsort((cols, rows) if by_row else (rows, cols))     # the last key is the primary one
    return rows[sigma], cols[sigma], P[sigma]


def coo2csr(rows, m: int, base: int = 0):
    return np.searchsorted(np.asarray(rows, np.int64) - base, np.arange(m + 1), side="left").astype(np.int64) + base


def csr2coo(off, base: int = 0):
    off = np.asarray(off, np.int64)
    return np.repeat(np.arange(off.size - 1, dtype=np.int64), np.diff(off)) + base


def _up(b: int) -> int:
    return (b + 255) // 256 * 256


def sort_scratch(nnz: int) -> int:
    """the radix sort's scratch: two key and two index buffers, the tile histograms, the digit totals"""
    return 4 * _up(4 * nnz) + _up(4 * 256 * -(-nnz // T.RT_TILE)) + _up(4 * 256)


def workspace(op: str, nnz: int) -> int:
    """csr2csc: the sort's scratch (the permutation is its last index buffer); coosort: that and the first sort's permutation"""
    return sort_scratch(nnz) + (_up(4 * nnz) if op == "coosort" else 0)
