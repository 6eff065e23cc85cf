"""oracle/spmm_coo_ref.py -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

Exact fixtures for the COO product C = alpha * op(A) * B + beta * C (spmm_coo.cu), in the manner of oracle/bell_ref.py.

A, B and C0 hold small integers, alpha and beta are powers of two (or 0 / +-1).  `check_exact` asserts that every partial sum stays
below 2^24, so the fp32 accumulator holds it whatever the summation order (atomics included), and that every output is an integer
below 2^24.  Any correct kernel then returns `reference` bit for bit, in fp32 and in fp64.

`walk` restates the row-sorted path of spmm_coo_sorted_kernel / spmm_coo_fixup_kernel in numpy (chunks of `chunk` entries, runs of
equal row index, the two carry slots per chunk, the fix-up in ascending chunk order, the rows that store nothing), so the CPU tests can
show that it computes the reference, writes every entry of C exactly once, and that the GPU test sizes land on every edge (`edges`).
"""
from __future__ import annotations

import ctypes as C

import numpy as np

from oracle import oracle as O


def params(lib=None) -> dict:
    if lib is None:
        from cudalibrarysamples_b200 import lib as _lib
        lib = _lib.shim()
    ch, pa, fo = C.c_int32(), C.c_int32(), C.c_int64()
    lib.b200spmm_coo_params(C.byref(ch), C.byref(pa), C.byref(fo))
    return dict(chunk=ch.value, panel=pa.value, flag_offset=fo.value)


def samples() -> dict:
    """spmm_coo and spmm_coo_batched: their data is the toy matrix of oracle.TOY / oracle.TOY_BATCHED (the COO samples store the same
    entries as spmm_csr / spmm_csr_batched, each batch with the row indices of spmm_coo_example.c:54); B and C column-major 4 x 3."""
    T, TB = O.TOY, O.TOY_BATCHED
    return {
        "spmm_coo": dict(rows=4, cols=4, n=3, row=T["coo_row"], col=T["csr_col"], val=T["val"], B=T["spmm_B"].T.ravel(),
                         C=T["spmm_C"].T.ravel()),
        "spmm_coo_batched": dict(rows=4, cols=4, n=3, batches=2, row=np.tile(T["coo_row"], 2), col=TB["csr_col"].ravel(),
                                 val=TB["val"].ravel(), B=TB["B"].ravel(), C=TB["C"].ravel()),
    }


# ------------------------------------------------------------------------------------------------ reference
def dense(rows, cols, row, col, val, base=0, transpose=False, dtype=np.int64):
    """the dense op(A); duplicate entries add up"""
    out = np.zeros((rows, cols), dtype)
    np.add.at(out, (np.asarray(row, np.int64) - base, np.asarray(col, np.int64) - base), np.asarray(val).astype(dtype))
    return out.T.copy() if transpose else out


def products(rows, cols, row, col, val, b, base=0, transpose=False, absolute=False):
    """int64 op(A) @ B (absolute: |op(A)| @ |B|, the largest partial sum any order can reach)"""
    d = dense(rows, cols, row, col, np.abs(val) if absolute else val, base, transpose)
    return d @ (np.abs(b) if absolute else np.asarray(b, np.int64))


def reference(rows, cols, row, col, val, b, c0, alpha, beta, base=0, transpose=False):
    """alpha * op(A) @ B + beta * C0, exact in fp64 (integers and powers of two); beta == 0 ignores C0"""
    out = alpha * products(rows, cols, row, col, val, b, base, transpose).astype(np.float64)
    if beta != 0:
        out = out + beta * np.asarray(c0, np.float64)
    return out


def check_exact(rows, cols, row, col, val, b, c0, alpha, beta, base=0, transpose=False):
    """every partial sum below 2^24, alpha / beta powers of two (or 0), every output an integer below 2^24"""
    for x in (alpha, beta):
        assert x == 0 or np.log2(abs(x)) == np.round(np.log2(abs(x)))
    s = products(rows, cols, row, col, val, b, base, transpose, absolute=True).astype(np.float64)
    bound = abs(alpha) * s + (abs(beta) * np.abs(np.asarray(c0, np.float64)) if beta != 0 else 0)
    assert (bound < (1 << 24)).all()
    ref = reference(rows, cols, row, col, val, b, c0, alpha, beta, base, transpose)
    assert (ref == np.round(ref)).all()


# ------------------------------------------------------------------------------------------------ the row-sorted walk
def walk(rows, row, col, val, b, c0, alpha, beta, chunk, base=0):
    """C of the row-sorted path, computed the way the kernels do, and how often each entry of C was written"""
    r = np.asarray(row, np.int64) - base
    c = np.asarray(col, np.int64) - base
    v = np.asarray(val, np.float64)
    b = np.asarray(b, np.float64)
    n = b.shape[1]
    nnz = r.size
    assert (np.diff(r) >= 0).all(), "the sorted path needs row-sorted entries"
    out = np.full((rows, n), np.nan)
    writes = np.zeros((rows, n), np.int64)
    c0 = np.asarray(c0, np.float64)

    def put(i, acc):
        out[i] = alpha * acc + (beta * c0[i] if beta != 0 else 0)
        writes[i] += 1

    def gap(lo, hi):
        for i in range(lo, hi):
            out[i] = beta * c0[i] if beta != 0 else 0
            writes[i] += 1
    if nnz == 0:
        gap(0, rows)
        return out, writes
    nchunks = -(-nnz // chunk)
    carry_row = np.full((nchunks, 2), -1, np.int64)
    carry_val = np.zeros((nchunks, 2, n))
    for k in range(nchunks):
        n0, n1 = k * chunk, min((k + 1) * chunk, nnz)
        gap((r[n0 - 1] if n0 > 0 else -1) + 1, r[n0])
        cur, acc, runs = r[n0], np.zeros(n), 0
        for e in range(n0, n1):
            if r[e] != cur:
                if runs == 0:
                    carry_row[k, 0], carry_val[k, 0] = cur, acc
                else:
                    put(cur, acc)
                gap(cur + 1, r[e])
                runs += 1
                cur, acc = r[e], np.zeros(n)
            acc = acc + v[e] * b[c[e]]
        s = 0 if runs == 0 else 1
        carry_row[k, s], carry_val[k, s] = cur, acc
        if k == nchunks - 1:
            gap(cur + 1, rows)
    flat_r, flat_v = carry_row.ravel(), carry_val.reshape(-1, n)
    live = np.flatnonzero(flat_r >= 0)
    for i, q in enumerate(live):                                 # the first slot of each row adds them all in ascending chunk order
        if i > 0 and flat_r[live[i - 1]] == flat_r[q]:
            continue
        acc = flat_v[q].copy()
        for q2 in live[i + 1:]:
            if flat_r[q2] != flat_r[q]:
                break
            acc = acc + flat_v[q2]
        put(flat_r[q], acc)
    return out, writes


def edges(rows, row, chunk, base=0) -> dict:
    """which edges of the chunk walk a row-sorted entry list reaches"""
    r = np.asarray(row, np.int64) - base
    nnz = r.size
    present = np.zeros(rows, bool)
    present[r] = True
    first_chunk, last_chunk = {}, {}
    for e, x in enumerate(r):
        first_chunk.setdefault(int(x), e // chunk)
        last_chunk[int(x)] = e // chunk
    span = {x: last_chunk[x] - first_chunk[x] + 1 for x in first_chunk}
    border_gap = any(r[k * chunk] - r[k * chunk - 1] > 1 for k in range(1, -(-nnz // chunk)))
    empty = np.flatnonzero(~present)
    return dict(nnz_mod=nnz % chunk if nnz else None, chunks=-(-nnz // chunk), max_span=max(span.values(), default=0),
                split_rows=sum(1 for s in span.values() if s > 1), empty_first=bool(rows and not present[0]),
                empty_last=bool(rows and not present[-1]), empty_middle=bool(((empty > r.min()) & (empty < r.max())).any()) if nnz else False,
                empty_across_border=bool(border_gap), all_empty=nnz == 0)


# ------------------------------------------------------------------------------------------------ generators
def sorted_rows(rows, counts):
    """row-sorted row indices: row i repeated counts[i] times"""
    return np.repeat(np.arange(rows, dtype=np.int32), np.asarray(counts, np.int64))


def values(nnz, kdim, crows, n, seed, lo=-2, hi=2):
    """int64 values, B (kdim x n) and C0 (crows x n, even) in [lo, hi]"""
    rng = np.random.default_rng(seed)
    v = rng.integers(lo, hi + 1, nnz, dtype=np.int64)
    b = rng.integers(lo, hi + 1, (kdim, n), dtype=np.int64)
    c0 = 2 * rng.integers(-3, 4, (crows, n), dtype=np.int64)
    return v, b, c0
