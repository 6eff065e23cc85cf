#!/usr/bin/env python
"""BSR SpMM, ours (b200spmm_bsr) against the closed library's cusparseSpMM on the same buffers, in one process (DESIGN.md 3.17).

C = A . V with A the softmaxed scores of block-sparse attention in BSR and V dense: the P . V half of the layer whose Q . K^T
scripts/sddmm_bsr_bench.py measures, on the same patterns (a sliding window of block columns plus global block-rows / block-columns,
and uniform random blocks at 10 % and 30 %).  Sizes: sequence length 4096 and 16384, bs 16 / 32 / 64 / 128, N (the head dimension)
64 and 128.  Types: f16 -> f16, f16 -> f32, bf16 -> bf16, bf16 -> f32, f32, f64.  Layouts: the attention one (V and O row-major) and
column-major.  Batches: 16 heads sharing one pattern.

Each call is timed with CUDA events after a warm-up (median of three windows).  Reported per case: us for ours (with the workspace the
shim passes, so the split walk) and for the closed library, TFLOP/s on 2 * bnnz * bs^2 * N * batch, the data-sheet bound that
applies (flops over the dense rate of the type, or bytes over 3.35 TB/s: A's values once, the B rows the pattern references, C), and
each side's largest error against fp64 relative to sum_k |a_ik| |b_kj|.  The card's name and power limit are read in the same run.
--status records the closed library's statuses of bufferSize / preprocess / SpMM over type x bs x op x order x batch layout.
usage: python scripts/spmm_bsr_bench.py [--quick] [--status] [--seq 4096 16384] [--no-heads] [--json out.json]"""
import argparse
import ctypes as C
import json
import os
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from cudalibrarysamples_b200 import cusparse_api as cs  # noqa: E402
from cudalibrarysamples_b200 import lib as _lib  # noqa: E402
from scripts.sddmm_bsr_bench import PEAK, PEAK_BYTES, card, pattern, timeit  # noqa: E402

DEV = torch.device("cuda:0")
ROW, COL = cs.CUSPARSE_ORDER_ROW, cs.CUSPARSE_ORDER_COL
NT, TR = cs.CUSPARSE_OPERATION_NON_TRANSPOSE, cs.CUSPARSE_OPERATION_TRANSPOSE
VT = {torch.float32: 0, torch.float64: 1, torch.float16: 2, torch.bfloat16: 14}
TYPES = [("f16-f16", torch.float16, torch.float16), ("f16-f32", torch.float16, torch.float32), ("bf16-bf16", torch.bfloat16, torch.bfloat16),
         ("bf16-f32", torch.bfloat16, torch.float32), ("f32", torch.float32, torch.float32), ("f64", torch.float64, torch.float64)]

# The classes b200spmm_bsr_route runs natively (DESIGN.md 3.17), as the predicate the CPU route test evaluates over
# (A / B type, C type, bs, N, M, order of B and C) with opB = N and row-major blocks.
NATIVE = ("lambda vt, cvt, bs, n, m, order: vt in (F16, BF16) and cvt in (vt, F32) and bs % 16 == 0 and bs <= 128 "
          "and 64 <= n <= 128 and (m >= 16384 or (bs >= 64 and m >= 4096))")


def operands(m, n, bs, bnnz, dt, ct, order, seed, batch=1):
    """softmax-like A values in [0, 1) (bnnz blocks per matrix), V (m x n) and a NaN-free C in the given order, batch matrices each"""
    g = torch.Generator(device=DEV).manual_seed(seed)
    vals = torch.rand(batch * bnnz * bs * bs, device=DEV, generator=g).to(dt)
    V = (torch.rand(batch, m, n, device=DEV, generator=g) * 2 - 1).to(dt)
    if order == COL:
        V = V.transpose(1, 2)
    return vals, V.contiguous(), torch.zeros(batch * m * n, dtype=ct, device=DEV)


def reference_error(off, col, vals, V, got, bs, order, nsample=8):
    """largest |c - fp64| / sum_k |a_ik| |b_kj| over up to nsample block-rows of the first matrix of the batch"""
    m = (off.numel() - 1) * bs
    n = V.shape[2] if order == ROW else V.shape[1]
    Vd = (V[0] if order == ROW else V[0].t()).double()
    Cd = got[:m * n].view(m, n) if order == ROW else got[:m * n].view(n, m).t()
    blocks = vals[:col.numel() * bs * bs].double().view(-1, bs, bs)
    offc = off.cpu().numpy()
    colc = col.cpu().numpy()
    rows = np.random.default_rng(0).permutation(len(offc) - 1)[:nsample]
    err = 0.0
    for r in rows:
        s, e = offc[r], offc[r + 1]
        ref = torch.zeros(bs, n, dtype=torch.float64, device=DEV)
        bound = torch.zeros_like(ref)
        for q in range(s, e):
            Vb = Vd[colc[q] * bs:(colc[q] + 1) * bs]
            ref += blocks[q] @ Vb
            bound += blocks[q].abs() @ Vb.abs()
        d = (Cd[r * bs:(r + 1) * bs].double() - ref).abs() / bound.clamp(min=1e-300)
        err = max(err, float(d.max()))
    return err


class Closed:
    """the closed library's cusparseSpMM on a BSR A, descriptors built once"""

    def __init__(self, m, n, bs, off, col, vals, V, Cb, order, ct, batch=1):
        self.api = cs.Api("cusparse")
        R = self.R = self.api.real
        self.h = self.api.cusparseCreate()
        ld = n if order == ROW else m
        self.matB = self.api.cusparseCreateDnMat(m, n, ld, V, order)
        self.matC = self.api.cusparseCreateDnMat(m, n, ld, Cb, order)
        d = C.c_void_p()
        bnnz = col.numel()
        assert R.cusparseCreateBsr(C.byref(d), C.c_int64(m // bs), C.c_int64(m // bs), C.c_int64(bnnz), C.c_int64(bs), C.c_int64(bs),
                                   C.c_void_p(off.data_ptr()), C.c_void_p(col.data_ptr()), C.c_void_p(vals.data_ptr()), 2, 2, 0,
                                   VT[vals.dtype], ROW) == 0
        self.matA = d
        self.status = 0
        if batch > 1:
            self.api.cusparseDnMatSetStridedBatch(self.matB, batch, m * n)
            self.api.cusparseDnMatSetStridedBatch(self.matC, batch, m * n)
            self.status = R.cusparseBsrSetStridedBatch(d, batch, C.c_int64(0), C.c_int64(0), C.c_int64(bnnz * bs * bs))
        self.ct = ct
        self.alpha, self.beta = (C.c_double(1.0), C.c_double(0.0)) if ct == 1 else (C.c_float(1.0), C.c_float(0.0))
        size = C.c_size_t(0)
        if self.status == 0:
            self.status = R.cusparseSpMM_bufferSize(self.h, NT, NT, C.byref(self.alpha), self.matA, self.matB, C.byref(self.beta),
                                                    self.matC, ct, 0, C.byref(size))
        self.buf = torch.empty(max(size.value, 16), dtype=torch.uint8, device=DEV)
        if self.status == 0:
            self.status = R.cusparseSpMM_preprocess(self.h, NT, NT, C.byref(self.alpha), self.matA, self.matB, C.byref(self.beta),
                                                    self.matC, ct, 0, C.c_void_p(self.buf.data_ptr()))

    def __call__(self):
        st = self.R.cusparseSpMM(self.h, NT, NT, C.byref(self.alpha), self.matA, self.matB, C.byref(self.beta), self.matC, self.ct, 0,
                                 C.c_void_p(self.buf.data_ptr()))
        assert st == 0, st

    def close(self):
        self.R.cusparseDestroySpMat(self.matA)
        self.api.cusparseDestroyDnMat(self.matB)
        self.api.cusparseDestroyDnMat(self.matC)
        self.api.cusparseDestroy(self.h)


def run_case(L, name, m, bs, n, dt, ctype, order, off_np, col_np, batch=1, seed=1, split=True):
    off = torch.tensor(off_np, dtype=torch.int32, device=DEV)
    col = torch.tensor(col_np, dtype=torch.int32, device=DEV)
    bnnz = int(col.numel())
    vals, V, ours_c = operands(m, n, bs, bnnz, dt, ctype, order, seed, batch)
    closed_c = torch.zeros_like(ours_c)
    f64 = dt == torch.float64
    one, zero = (C.c_double(1.0), C.c_double(0.0)) if f64 else (C.c_float(1.0), C.c_float(0.0))
    sbk, sbj = (n, 1) if order == ROW else (1, m)
    wsb = L.b200spmm_bsr_workspace_bytes(VT[dt], m, n, bs, bnnz, batch) if split else 0
    ws = torch.empty(max(wsb, 16), dtype=torch.uint8, device=DEV)
    stream = torch.cuda.current_stream().cuda_stream

    def ours():
        rc = L.b200spmm_bsr(stream, VT[dt], VT[ctype], m, m, n, bs, bnnz, off.data_ptr(), col.data_ptr(), vals.data_ptr(), 0, 1,
                            C.addressof(one), C.addressof(zero), 0, V.data_ptr(), sbk, sbj, ours_c.data_ptr(), n if order == ROW else m,
                            1 if order == ROW else 0, batch, 0, 0, bnnz * bs * bs if batch > 1 else 0, m * n if batch > 1 else 0,
                            m * n if batch > 1 else 0,
                            ws.data_ptr() if split else None, wsb)
        assert rc == 0, rc
    ct = 1 if f64 else 0
    closed = Closed(m, n, bs, off, col, vals, V, closed_c, order, ct, batch)
    row = dict(case=name, m=m, bs=bs, n=n, type=f"{str(dt)[6:]}->{str(ctype)[6:]}", order="row" if order == ROW else "col", batch=batch,
               bnnz=bnnz, path="tensor" if L.b200spmm_bsr_path(VT[dt], bs, 1, vals.data_ptr(), V.data_ptr(), sbk, sbj, batch,
                                                              bnnz * bs * bs, m * n if batch > 1 else 0) else "cuda-core")
    t_ours = timeit(ours)
    row["us_ours"] = t_ours * 1e6
    row["err_ours"] = reference_error(off, col, vals, V, ours_c, bs, order)
    if closed.status == 0:
        t_cl = timeit(closed)
        row["us_closed"] = t_cl * 1e6
        row["err_closed"] = reference_error(off, col, vals, V, closed_c, bs, order)
        row["speedup"] = t_cl / t_ours
    else:
        row["closed_status"] = closed.status
    closed.close()
    flops = 2.0 * bnnz * bs * bs * n * batch
    es = vals.element_size()
    used_rows = len(np.unique(col_np)) * bs
    bytes_ = bnnz * bs * bs * es + (used_rows * n * es + m * n * ours_c.element_size()) * batch + (m // bs + 1 + bnnz) * 4
    t_flop, t_byte = flops / PEAK[dt], bytes_ / PEAK_BYTES
    row["tflops_ours"] = flops / t_ours / 1e12
    row["bound"] = "flops" if t_flop >= t_byte else "bytes"
    row["bound_us"] = max(t_flop, t_byte) * 1e6
    return row


def status_grid():
    """which combinations the closed library accepts: statuses of bufferSize / preprocess / SpMM over type x bs x opB x order x
    block order x batch layout"""
    R = _lib.real()
    api = cs.Api("cusparse")
    h = api.cusparseCreate()
    out = []
    m, n = 256, 64
    buf = torch.empty(1 << 24, dtype=torch.uint8, device=DEV)

    def one(dt, ctype, compute, bs, opB, ob, oc, oa=ROW, batch=1, shared="", alg=0):
        nb = m // bs
        off = torch.arange(0, nb + 1, dtype=torch.int32, device=DEV).repeat(batch)       # a copy per matrix, whether shared or not
        col = torch.arange(0, nb, dtype=torch.int32, device=DEV).repeat(batch)
        vals = torch.zeros(batch * nb * bs * bs, dtype=dt, device=DEV)
        B = torch.zeros(batch * m * n, dtype=dt, device=DEV)
        Cm = torch.zeros(batch * m * n, dtype=ctype, device=DEV)
        br, bc = (m, n) if opB == NT else (n, m)
        mB = api.cusparseCreateDnMat(br, bc, bc if ob == ROW else br, B, ob)
        mC = api.cusparseCreateDnMat(m, n, n if oc == ROW else m, Cm, oc)
        d = C.c_void_p()
        st = R.cusparseCreateBsr(C.byref(d), C.c_int64(nb), C.c_int64(nb), C.c_int64(nb), C.c_int64(bs), C.c_int64(bs),
                                 C.c_void_p(off.data_ptr()), C.c_void_p(col.data_ptr()), C.c_void_p(vals.data_ptr()), 2, 2, 0, VT[dt], oa)
        sts = {"create": st}
        if st == 0:
            if batch > 1:
                if "B" not in shared:
                    api.cusparseDnMatSetStridedBatch(mB, batch, m * n)
                api.cusparseDnMatSetStridedBatch(mC, batch, m * n)
                sts["setStridedBatch"] = R.cusparseBsrSetStridedBatch(d, batch, C.c_int64(0 if "o" in shared else nb + 1),
                                                                      C.c_int64(0 if "c" in shared else nb),
                                                                      C.c_int64(0 if "v" in shared else nb * bs * bs))
            al, be = (C.c_double(1), C.c_double(0)) if compute == 1 else (C.c_float(1), C.c_float(0))
            size = C.c_size_t(0)
            sts["bufferSize"] = R.cusparseSpMM_bufferSize(h, NT, opB, C.byref(al), d, mB, C.byref(be), mC, compute, alg, C.byref(size))
            if sts["bufferSize"] == 0 and size.value <= buf.numel():
                sts["preprocess"] = R.cusparseSpMM_preprocess(h, NT, opB, C.byref(al), d, mB, C.byref(be), mC, compute, alg,
                                                              C.c_void_p(buf.data_ptr()))
                sts["spmm"] = R.cusparseSpMM(h, NT, opB, C.byref(al), d, mB, C.byref(be), mC, compute, alg, C.c_void_p(buf.data_ptr()))
            torch.cuda.synchronize()
            R.cusparseDestroySpMat(d)
        api.cusparseDestroyDnMat(mB)
        api.cusparseDestroyDnMat(mC)
        return sts

    def emit(**kw):
        out.append(kw)
        print(json.dumps(kw), flush=True)
    types = [(torch.float16, torch.float16, 0), (torch.float16, torch.float32, 0), (torch.bfloat16, torch.bfloat16, 0),
             (torch.bfloat16, torch.float32, 0), (torch.float32, torch.float32, 0), (torch.float64, torch.float64, 1),
             (torch.float16, torch.float16, 2)]
    for dt, ctype, compute in types:
        t = f"{str(dt)[6:]}->{str(ctype)[6:]}/{compute}"
        for bs in (1, 2, 4, 8, 16, 32, 64, 128):
            for opB in (NT, TR):
                for ob in (ROW, COL):
                    for oc in (ROW, COL):
                        emit(type=t, bs=bs, opB=opB, orderB=ob, orderC=oc, **one(dt, ctype, compute, bs, opB, ob, oc))
        for bs in (4, 16):
            emit(type=t, bs=bs, orderA="col", **one(dt, ctype, compute, bs, NT, ROW, ROW, oa=COL))
            emit(type=t, bs=bs, alg="BSR_ALG1", **one(dt, ctype, compute, bs, NT, ROW, ROW, alg=14))
            for shared in ("", "oc", "ocv", "B"):
                emit(type=t, bs=bs, batch=4, shared=shared or "-", **one(dt, ctype, compute, bs, NT, ROW, ROW, batch=4, shared=shared))
    api.cusparseDestroy(h)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--quick", action="store_true")
    ap.add_argument("--status", action="store_true", help="also print the closed library's status grid")
    ap.add_argument("--seq", type=int, nargs="+", default=[4096, 16384], help="sequence lengths")
    ap.add_argument("--no-heads", action="store_true", help="skip the 16-head batches")
    ap.add_argument("--json")
    args = ap.parse_args()
    L = _lib.shim()
    name = card()
    print(f"# card: {name}", flush=True)
    rows = []
    t0 = time.time()
    if args.status:
        status_grid()
    for seq in ([4096] if args.quick else args.seq):
        for kind in ("window", "rand10", "rand30"):
            for bs in (16, 32, 64, 128):
                off, col = pattern(kind, seq // bs, seed=bs)
                for n in (64, 128):
                    for tname, dt, ctype in TYPES:
                        for order in (ROW, COL):
                            if args.quick and (n == 128 or kind == "rand30" or order == COL):
                                continue
                            rows.append(run_case(L, kind, seq, bs, n, dt, ctype, order, off, col))
                            print(json.dumps(rows[-1]), flush=True)
    for tname, dt, ctype in ([] if args.no_heads else TYPES):
        for bs in (16, 64):
            off, col = pattern("window", 4096 // bs, seed=bs)
            rows.append(run_case(L, "window-16heads", 4096, bs, 64, dt, ctype, ROW, off, col, batch=16))
            print(json.dumps(rows[-1]), flush=True)
    print(f"# {len(rows)} cases in {time.time() - t0:.0f} s on {name}", flush=True)
    if args.json:
        with open(args.json, "w") as f:
            json.dump(dict(card=name, rows=rows), f, indent=1)


if __name__ == "__main__":
    main()
