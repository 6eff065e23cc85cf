"""oracle/bell_ref.py -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

Exact fixtures for the Blocked-ELL product C = alpha * A * B + beta * C (spmm_bell.cu), in the manner of oracle/sddmm_ref.py.

Format (cuSPARSE/dense2sparse_blockedell, spmm_blockedell): A is rows x cols in bs x bs blocks; col_ind is (rows / bs) x (ell_cols / bs)
block columns, row-major, -1 for an empty slot anywhere in a block-row; values is rows x ell_cols, row-major, row r holding its
block-row's blocks side by side.

A and B hold small integers, alpha and beta are powers of two (or 0 / +-1), C0 even integers.  `check_exact` asserts that every partial
sum stays below 2^24 (the fp32 accumulator holds it whatever the summation order) and that every output is an integer the output type
holds exactly: |v| <= 2048 for fp16, <= 256 for bf16, < 2^24 for fp32.  Any correct kernel then returns `reference` bit for bit.
"""
from __future__ import annotations

import ctypes as C
import json
import os

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SAMPLES = os.path.join(ROOT, "tests", "golden", "bell_samples.json")
OUT_LIMIT = {"f16": 2048, "bf16": 256, "f32": (1 << 24) - 1}      # the largest integer magnitude each output type holds
SCALARS = [(1.0, 0.0), (-1.0, 1.0), (2.0, 0.5), (-2.0, -2.0)]      # (alpha, beta); beta == 0 is run on a NaN-filled C


def samples() -> dict:
    """spmm_blockedell's inputs and golden (column-major B and C), and dense2sparse_blockedell's dense matrix with its Blocked-ELL arrays"""
    with open(SAMPLES) as f:
        return json.load(f)


def params(lib=None) -> dict:
    if lib is None:
        from cudalibrarysamples_b200 import lib as _lib
        lib = _lib.shim()
    t, s, r = C.c_int32(), C.c_int32(), C.c_int32()
    lib.b200spmm_bell_params(C.byref(t), C.byref(s), C.byref(r))
    return dict(n_tile=t.value, stages=s.value, max_rows_per_cta=r.value)


# ------------------------------------------------------------------------------------------------ converters
def to_dense(rows, cols, bs, col_ind, values, base=0, dtype=np.int64):
    """the dense rows x cols matrix of a Blocked-ELL A; empty slots are skipped, their values never looked at"""
    ci = np.asarray(col_ind, np.int64).reshape(rows // bs, -1)
    v = np.asarray(values).reshape(rows, -1)
    out = np.zeros((rows, cols), dtype)
    for br in range(ci.shape[0]):
        for j, c in enumerate(ci[br]):
            if c == -1:
                continue
            c -= base
            out[br * bs:(br + 1) * bs, c * bs:(c + 1) * bs] += v[br * bs:(br + 1) * bs, j * bs:(j + 1) * bs].astype(dtype)
    return out


def from_dense(dense, bs, ell_cols=None, base=0):
    """(col_ind, values) of a dense matrix: the non-zero blocks of each block-row in ascending block column, then -1 slots (zero
    values) up to ell_cols (default: the widest block-row)"""
    dense = np.asarray(dense)
    rows, cols = dense.shape
    nbr, nbc = rows // bs, cols // bs
    live = [[c for c in range(nbc) if dense[br * bs:(br + 1) * bs, c * bs:(c + 1) * bs].any()] for br in range(nbr)]
    eb = max((len(x) for x in live), default=0) if ell_cols is None else ell_cols // bs
    ci = np.full((nbr, eb), -1, np.int64)
    vals = np.zeros((rows, eb * bs), dense.dtype)
    for br, cs in enumerate(live):
        for j, c in enumerate(cs):
            ci[br, j] = c + base
            vals[br * bs:(br + 1) * bs, j * bs:(j + 1) * bs] = dense[br * bs:(br + 1) * bs, c * bs:(c + 1) * bs]
    return ci, vals


def to_scipy(rows, cols, bs, col_ind, values, base=0):
    """the same matrix as a scipy BSR matrix (blocks in slot order, empty slots dropped)"""
    import scipy.sparse as sp
    ci = np.asarray(col_ind, np.int64).reshape(rows // bs, -1)
    v = np.asarray(values, np.float64).reshape(rows, -1)
    indptr, indices, data = [0], [], []
    for br in range(ci.shape[0]):
        for j, c in enumerate(ci[br]):
            if c != -1:
                indices.append(c - base)
                data.append(v[br * bs:(br + 1) * bs, j * bs:(j + 1) * bs])
        indptr.append(len(indices))
    data = np.array(data).reshape(-1, bs, bs) if data else np.zeros((0, bs, bs))
    return sp.bsr_matrix((data, np.array(indices, np.int64), np.array(indptr, np.int64)), shape=(rows, cols))


# ------------------------------------------------------------------------------------------------ generators and reference
def structure(nbr, nbc, eb, live_counts, seed, base=0):
    """(nbr, eb) block columns: block-row i stores live_counts[i % len] distinct random block columns at random slots (so -1 slots
    fall first, in the middle and last), the rest -1"""
    rng = np.random.default_rng(seed)
    ci = np.full((nbr, eb), -1, np.int64)
    for br in range(nbr):
        k = min(live_counts[br % len(live_counts)], eb, nbc)
        slots = np.sort(rng.choice(eb, k, replace=False))
        ci[br, slots] = rng.choice(nbc, k, replace=False) + base
    return ci


def values(rows, ell_cols, cols, n, seed, lo=-1, hi=1):
    """int64 A values (rows x ell_cols), B (cols x n) and C0 (rows x n, even) in [lo, hi]"""
    rng = np.random.default_rng(seed)
    a = rng.integers(lo, hi + 1, (rows, ell_cols), dtype=np.int64)
    b = rng.integers(lo, hi + 1, (cols, n), dtype=np.int64)
    c0 = 2 * rng.integers(-3, 4, (rows, n), dtype=np.int64)
    return a, b, c0


def products(rows, cols, bs, col_ind, a, b, base=0, absolute=False):
    """int64 A @ B (absolute: |A| @ |B|, the largest partial sum any order can reach)"""
    d = to_dense(rows, cols, bs, col_ind, np.abs(a) if absolute else a, base)
    return d @ (np.abs(b) if absolute else b)


def reference(rows, cols, bs, col_ind, a, b, c0, alpha, beta, base=0):
    """alpha * A @ B + beta * C0, exact in fp64 (integers and powers of two)"""
    out = alpha * products(rows, cols, bs, col_ind, a, b, base).astype(np.float64)
    if beta != 0:
        out = out + beta * np.asarray(c0, np.float64)
    return out


def check_exact(rows, cols, bs, col_ind, a, b, c0, alpha, beta, out_kind, base=0):
    """every partial sum below 2^24, and every output an integer that `out_kind` ("f16", "bf16", "f32") holds exactly"""
    s = products(rows, cols, bs, col_ind, a, b, base, absolute=True)
    assert (s < (1 << 24)).all()
    for x in (alpha, beta):
        assert x == 0 or np.log2(abs(x)) == np.round(np.log2(abs(x)))
    ref = reference(rows, cols, bs, col_ind, a, b, c0, alpha, beta, base)
    bound = np.abs(alpha) * s + (np.abs(beta) * np.abs(np.asarray(c0, np.float64)) if beta != 0 else 0)
    assert (bound < (1 << 24)).all()
    assert (ref == np.round(ref)).all() and (np.abs(ref) <= OUT_LIMIT[out_kind]).all()
