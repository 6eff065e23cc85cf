#!/usr/bin/env python
"""Transposed CSR SpMM, ours (b200spmm_csr_t) against the closed library's cusparseSpMM with opA = TRANSPOSE on the same buffers, in
one process (DESIGN.md 3.22).

C = A^T . B with A a rows x cols CSR matrix: the backward pass of a graph layer (A^T G on the forward pass's pattern).  Matrices:
R-MAT 1M x 1M with 16 per row (skewed columns: the hub rows of A^T), uniform 2M x 2M with 16 per row, and the 5-point 8192^2 stencil
(a symmetric pattern).  N 32, 64, 128, 256; B and C both row-major and both column-major, opB = N; types fp32, fp64, fp16 and bf16
(C of A's type, fp32 compute for the 16-bit ones).

Reported per case, each timed with CUDA events after a warm-up (median of three windows): the plan build alone (`plan_us`), our call
with a trusted plan (`us_trusted`: the value gather and the opA = N kernels, what cusparseSpMM runs after cusparseSpMM_preprocess), our
call that rebuilds the plan (`us_rebuild`: a call without preprocess), the closed library's call after its preprocess (`us_closed`), the
speed-ups over it, and the largest difference between ours and the closed library relative to sum_k |a_ki| |b_kj| over sampled
columns (the closed library's transpose is not deterministic: no bit-for-bit comparison).  The card's name and power limit are read
in the same run.
usage: python scripts/spmm_csr_t_bench.py [--quick] [--json out.json]"""
import argparse
import ctypes as C
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from cudalibrarysamples_b200 import cusparse_api as cs  # noqa: E402
from cudalibrarysamples_b200 import lib as _lib  # noqa: E402
from cudalibrarysamples_b200 import workloads as W  # noqa: E402
from scripts.sddmm_bsr_bench import card, timeit  # noqa: E402

DEV = torch.device("cuda:0")
ROW, COL = cs.CUSPARSE_ORDER_ROW, cs.CUSPARSE_ORDER_COL
NT, TR = cs.CUSPARSE_OPERATION_NON_TRANSPOSE, cs.CUSPARSE_OPERATION_TRANSPOSE
VT = {torch.float32: 0, torch.float64: 1, torch.float16: 2, torch.bfloat16: 14}
TYPES = (torch.float32, torch.float64, torch.float16, torch.bfloat16)
MATRICES = ("rmat1m", "uniform2m", "stencil8192")
TOL = {torch.float32: 1e-5, torch.float64: 1e-13, torch.float16: 2e-2, torch.bfloat16: 1e-1}

# The classes b200spmm_csr_t_route runs natively (DESIGN.md 3.22), as the predicate the CPU route test evaluates over (trusted plan,
# opB (0 = N), A / B type, C type, N, rows, nnz, order of B, order of C): every case measured in a class ran at least at parity with
# the closed library.  Only opB = N was measured, so opB = T is forwarded.  16-bit: a trusted plan everywhere, a rebuilt one column-major or from N = 128; fp32 / fp64: column-major from
# N = 64 (R-MAT 1M lost at N = 32 and row-major at every N).  The 5-point 8192^2 stencil (5 per row, N = 32 only: fp64 and larger N do
# not fit beside the closed library's operands) stays outside: fp32 lost there (0.68x - 0.81x), and a density measured on one matrix
# does not make a class.
NATIVE = ("lambda trusted, opb, vt, cvt, n, m, nnz, ob, oc: opb == 0 and 1 << 20 <= m <= 2 << 20 and 16 * m <= nnz < 17 * m and 32 <= n <= 256 "
          "and ob == oc and cvt == vt and ((vt in (2, 14) and (trusted or oc == 1 or n >= 128)) or (vt in (0, 1) and oc == 1 and n >= 64))")


def matrix(name):
    """(rows, cols, off, col, fp32 values) on the device, base 0, sorted columns"""
    if name == "rmat1m":
        rows = 1 << 20
        off, col, val = W.rmat_csr(rows, avg_nnz=16, seed=42, val_seed=43, dtype=torch.float32)
    elif name == "uniform2m":
        rows = 2 << 20
        g = torch.Generator(device=DEV).manual_seed(5)
        col = torch.randint(0, rows, (rows * 16,), device=DEV, generator=g, dtype=torch.int32)
        col = col.view(rows, 16).sort(dim=1).values.reshape(-1).contiguous()
        off = torch.arange(0, rows * 16 + 1, 16, device=DEV, dtype=torch.int32)
        val = torch.rand(rows * 16, device=DEV, generator=g, dtype=torch.float32) * 2 - 1
    else:
        off, col, val = W.stencil5_csr(8192)
        rows = off.numel() - 1
    return rows, rows, off.int().contiguous(), col.int().contiguous(), val.float().contiguous()


class Closed:
    """the closed library's cusparseSpMM with opA = TRANSPOSE, descriptors and buffer built once, preprocess run once"""

    def __init__(self, rows, cols, n, off, col, vals, Bs, Cb, order, ct):
        self.api = cs.Api("cusparse")
        R = self.R = self.api.real
        self.h = self.api.cusparseCreate()
        self.matB = self.api.cusparseCreateDnMat(rows, n, n if order == ROW else rows, Bs, order)
        self.matC = self.api.cusparseCreateDnMat(cols, n, n if order == ROW else cols, Cb, order)
        d = C.c_void_p()
        assert R.cusparseCreateCsr(C.byref(d), C.c_int64(rows), C.c_int64(cols), C.c_int64(col.numel()), C.c_void_p(off.data_ptr()),
                                   C.c_void_p(col.data_ptr()), C.c_void_p(vals.data_ptr()), 2, 2, 0, VT[vals.dtype]) == 0
        self.matA, self.ct = d, ct
        self.alpha, self.beta = (C.c_double(1), C.c_double(0)) if ct == 1 else (C.c_float(1), C.c_float(0))
        size = C.c_size_t(0)
        self.status = R.cusparseSpMM_bufferSize(self.h, TR, NT, C.byref(self.alpha), self.matA, self.matB, C.byref(self.beta), self.matC,
                                                ct, 0, C.byref(size))
        self.buf = torch.empty(max(size.value, 16), dtype=torch.uint8, device=DEV)
        if self.status == 0:
            self.status = R.cusparseSpMM_preprocess(self.h, TR, NT, C.byref(self.alpha), self.matA, self.matB, C.byref(self.beta),
                                                    self.matC, ct, 0, C.c_void_p(self.buf.data_ptr()))

    def __call__(self):
        st = self.R.cusparseSpMM(self.h, TR, NT, C.byref(self.alpha), self.matA, self.matB, C.byref(self.beta), self.matC, self.ct, 0,
                                 C.c_void_p(self.buf.data_ptr()))
        assert st == 0, st

    def close(self):
        self.R.cusparseDestroySpMat(self.matA)
        self.api.cusparseDestroyDnMat(self.matB)
        self.api.cusparseDestroyDnMat(self.matC)
        self.api.cusparseDestroy(self.h)


def difference(ours, closed, bound):
    return float(((ours.double() - closed.double()).abs() / bound.clamp(min=1e-300)).max())


def run_case(L, name, rows, cols, off, col, val32, n, dt, order, seed=1):
    nnz = col.numel()
    vals = val32.to(dt)
    g = torch.Generator(device=DEV).manual_seed(seed)
    Bop = (torch.rand(rows, n, device=DEV, generator=g) * 2 - 1).to(dt)          # B, rows x n
    Bs = Bop.contiguous() if order == ROW else Bop.t().contiguous()
    ours_c = torch.zeros(cols * n, dtype=dt, device=DEV)
    closed_c = torch.zeros_like(ours_c)
    ct = 1 if dt == torch.float64 else 0
    one, zero = (C.c_double(1), C.c_double(0)) if ct == 1 else (C.c_float(1), C.c_float(0))
    sbk, sbj = (n, 1) if order == ROW else (1, rows)
    ldc = n if order == ROW else cols
    wsb = L.b200spmm_csr_t_workspace_bytes(VT[dt], rows, cols, n, nnz, sbk, sbj)
    ws = torch.empty(wsb, dtype=torch.uint8, device=DEV)
    stream = torch.cuda.current_stream().cuda_stream

    def ours(plan_valid):
        rc = L.b200spmm_csr_t(stream, VT[dt], VT[dt], rows, cols, n, nnz, off.data_ptr(), col.data_ptr(), vals.data_ptr(), 0,
                              C.addressof(one), C.addressof(zero), 0, Bs.data_ptr(), sbk, sbj, ours_c.data_ptr(), ldc,
                              1 if order == ROW else 0, plan_valid, ws.data_ptr(), wsb)
        assert rc == 0, rc

    def plan():
        assert L.b200spmm_csr_t_plan(stream, rows, cols, nnz, off.data_ptr(), col.data_ptr(), 0, ws.data_ptr(), wsb) == 0

    row = dict(case=name, rows=rows, nnz=nnz, n=n, type=str(dt)[6:], order="row" if order == ROW else "col", ws_mb=wsb / 2 ** 20)
    row["plan_us"] = timeit(plan) * 1e6
    row["us_rebuild"] = timeit(lambda: ours(0)) * 1e6
    row["us_trusted"] = timeit(lambda: ours(1)) * 1e6
    closed = Closed(rows, cols, n, off, col, vals, Bs, closed_c, order, ct)
    row["closed_ws_mb"] = closed.buf.numel() / 2 ** 20
    if closed.status == 0:
        row["us_closed"] = timeit(closed) * 1e6
        row["speedup_trusted"] = row["us_closed"] / row["us_trusted"]
        row["speedup_rebuild"] = row["us_closed"] / row["us_rebuild"]
        # |A|^T |B| bounds every rounding of either side: over 64 sampled columns of A (rows of C) and the longest one
        lens = torch.bincount(col.long(), minlength=cols)
        pick = torch.unique(torch.cat([torch.randperm(cols, device=DEV, generator=g)[:64], lens.argmax().view(1)]))
        sel = torch.isin(col.long(), pick).nonzero().view(-1)
        r_of = torch.searchsorted(off[1:].long(), sel, right=True)
        where = torch.searchsorted(pick, col.long()[sel])
        bound = torch.zeros(pick.numel(), n, dtype=torch.float64, device=DEV)
        bound.index_add_(0, where, vals[sel].double().abs()[:, None] * Bop[r_of].double().abs())
        oc = ours_c.view(cols, n) if order == ROW else ours_c.view(n, cols).t()
        cc = closed_c.view(cols, n) if order == ROW else closed_c.view(n, cols).t()
        row["diff"] = difference(oc[pick], cc[pick], bound)
        row["ok"] = row["diff"] <= TOL[dt]
    else:
        row["closed_status"] = closed.status
    closed.close()
    # what the shim's route decides for this class, trusted plan / rebuilt plan: the predicate above, printed beside the speed-ups
    native = eval(NATIVE)
    o = 2 if order == ROW else 1
    row["routed_trusted"] = bool(native(True, 0, VT[dt], VT[dt], n, rows, nnz, o, o))
    row["routed_rebuild"] = bool(native(False, 0, VT[dt], VT[dt], n, rows, nnz, o, o))
    return row


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--quick", action="store_true")
    ap.add_argument("--json")
    ap.add_argument("--matrices", default=",".join(MATRICES))
    ap.add_argument("--ns", default="32,64,128,256")
    a = ap.parse_args()
    L = _lib.shim()
    print(f"card: {card()}", flush=True)
    out = []
    mats = MATRICES[:1] if a.quick else a.matrices.split(",")
    ns = (64,) if a.quick else tuple(int(x) for x in a.ns.split(","))
    for name in mats:
        rows, cols, off, col, val = matrix(name)
        for dt in TYPES:
            for n in ns:
                for order in (ROW, COL):
                    try:
                        r = run_case(L, name, rows, cols, off, col, val, n, dt, order)
                    except torch.OutOfMemoryError:                   # both sides' operands and buffers exceed the card
                        r = dict(case=name, n=n, type=str(dt)[6:], order="row" if order == ROW else "col", oom=True)
                    out.append(r)
                    print(json.dumps(r), flush=True)
                    torch.cuda.empty_cache()
        del off, col, val
    if a.json:
        with open(a.json, "w") as f:
            json.dump({"card": card(), "rows": out}, f, indent=1)


if __name__ == "__main__":
    main()
