#!/usr/bin/env python
"""BSR SDDMM, ours (b200sddmm_bsr) against the closed library's cusparseSDDMM on the same buffers, in one process (DESIGN.md 3.16).

Patterns: a sliding window of block columns plus a few global block-rows / block-columns (the Longformer / BigBird shape), uniform
random blocks at 10 % and 30 %, and the sddmm_bsr sample itself.  Sizes: sequence length 4096 and 16384, bs 16 / 32 / 64 / 128, K 64
and 128.  Types: f16 -> f16, f16 -> f32, bf16 -> f32, f32, f64.  Layouts: the sample's (A M x K row-major, B K x N row-major, N / N) and
the attention one (B N x K row-major, opB = T).  Batches: 16 heads sharing one pattern, where the closed library takes that layout.

Each call is timed with CUDA events after a warm-up (median of several windows).  Reported per case: us for ours and the closed
library, TFLOP/s on 2 * bnnz * bs^2 * K * batch, which data-sheet bound applies (flops over the dense rate of the type, or bytes
over 3.35 TB/s), and each side's largest error against fp64 relative to the dot-product bound sum_k |a_ik| |b_kj|.  The card's name
and power limit are read in the same run.
usage: python scripts/sddmm_bsr_bench.py [--quick] [--status] [--seq 4096 16384] [--no-heads] [--json out.json]"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from cudalibrarysamples_b200 import cusparse_api as cs  # noqa: E402
from cudalibrarysamples_b200 import lib as _lib  # noqa: E402

DEV = torch.device("cuda:0")
ROW, COL = cs.CUSPARSE_ORDER_ROW, cs.CUSPARSE_ORDER_COL
NT, TR = cs.CUSPARSE_OPERATION_NON_TRANSPOSE, cs.CUSPARSE_OPERATION_TRANSPOSE
PEAK = {torch.float16: 989e12, torch.bfloat16: 989e12, torch.float32: 67e12, torch.float64: 34e12}   # H100 SXM data sheet, dense
PEAK_BYTES = 3.35e12
VT = {torch.float32: 0, torch.float64: 1, torch.float16: 2, torch.bfloat16: 14}
TYPES = [("f16-f16", torch.float16, torch.float16), ("f16-f32", torch.float16, torch.float32), ("bf16-f32", torch.bfloat16, torch.float32),
         ("f32", torch.float32, torch.float32), ("f64", torch.float64, torch.float64)]


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name(0)


def pattern(kind, nb, seed):
    """block offsets and block columns (int32, base 0, ascending columns per block-row) of an nb x nb block pattern"""
    rng = np.random.default_rng(seed)
    if kind == "window":                        # +-2 block columns around the diagonal, 2 global block-rows and block-columns
        mask = np.zeros((nb, nb), bool)
        for d in range(-2, 3):
            idx = np.arange(max(0, -d), min(nb, nb - d))
            mask[idx, idx + d] = True
        mask[:2, :] = True
        mask[:, :2] = True
    else:
        mask = rng.random((nb, nb)) < {"rand10": 0.10, "rand30": 0.30}[kind]
    off = np.concatenate([[0], np.cumsum(mask.sum(1))]).astype(np.int32)
    col = np.nonzero(mask)[1].astype(np.int32)
    return off, col


def operands(m, n, k, dt, layout, seed, batch=1):
    g = torch.Generator(device=DEV).manual_seed(seed)
    A = (torch.rand(batch, m, k, device=DEV, generator=g) * 2 - 1).to(dt)
    if layout == "sample":                       # B K x N row-major, opB = N
        B = (torch.rand(batch, k, n, device=DEV, generator=g) * 2 - 1).to(dt)
    else:                                        # B N x K row-major, opB = T
        B = (torch.rand(batch, n, k, device=DEV, generator=g) * 2 - 1).to(dt)
    return A.contiguous(), B.contiguous()


def reference_error(off, col, vals, A, B, bs, layout, nsample=2048):
    """largest |c - fp64| / sum_k |a||b| over up to nsample stored blocks of the first matrix of the batch"""
    bnnz = col.numel()
    rows = torch.repeat_interleave(torch.arange(off.numel() - 1, device=DEV), (off[1:] - off[:-1]).long())
    pick = torch.randperm(bnnz, device=DEV)[:nsample]
    Ad = A[0].double().view(-1, bs, A.shape[-1])[rows[pick]]                           # (s, bs, K)
    Bt = B[0].double() if layout != "sample" else B[0].double().t()
    Bd = Bt.reshape(-1, bs, Bt.shape[-1])[col[pick].long()]                           # (s, bs, K)
    ref = torch.bmm(Ad, Bd.transpose(1, 2))
    bound = torch.bmm(Ad.abs(), Bd.abs().transpose(1, 2)).clamp(min=1e-300)
    got = vals.view(-1, bnnz, bs, bs)[0][pick].double()
    return float(((got - ref).abs() / bound).max())


def timeit(fn, budget=0.02):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record(); fn(); e.record(); torch.cuda.synchronize()
    one = max(s.elapsed_time(e) / 1e3, 1e-6)
    reps = int(min(200, max(3, budget / one)))
    ts = []
    for _ in range(3):
        s.record()
        for _ in range(reps):
            fn()
        e.record()
        torch.cuda.synchronize()
        ts.append(s.elapsed_time(e) / 1e3 / reps)
    return float(np.median(ts))


class Closed:
    """the closed library's cusparseSDDMM with descriptors built once (sddmm_bsr_example.c's call sequence)"""

    def __init__(self, m, n, k, bs, off, col, vals, A, B, layout, ct, batch=1, share_pattern=True):
        self.api = cs.Api("cusparse")
        R = self.api.real
        self.R = R
        self.h = self.api.cusparseCreate()
        self.opB = NT if layout == "sample" else TR
        self.matA = self.api.cusparseCreateDnMat(m, k, k, A, ROW)
        br, bc = (k, n) if layout == "sample" else (n, k)
        self.matB = self.api.cusparseCreateDnMat(br, bc, bc, B, ROW)
        d = C.c_void_p()
        bnnz = col.numel() // (1 if share_pattern else batch)
        st = R.cusparseCreateBsr(C.byref(d), C.c_int64(m // bs), C.c_int64(n // bs), C.c_int64(bnnz), C.c_int64(bs), C.c_int64(bs),
                                 C.c_void_p(off.data_ptr()), C.c_void_p(col.data_ptr()), C.c_void_p(vals.data_ptr()), 2, 2, 0, VT[vals.dtype],
                                 ROW)
        assert st == 0, st
        self.matC = d
        self.status = 0
        if batch > 1:
            self.api.cusparseDnMatSetStridedBatch(self.matA, batch, m * k)
            self.api.cusparseDnMatSetStridedBatch(self.matB, batch, n * k)
            self.status = R.cusparseBsrSetStridedBatch(d, batch, C.c_int64(0), C.c_int64(0 if share_pattern else bnnz),
                                                       C.c_int64(bnnz * bs * bs))
        self.ct = ct
        self.alpha, self.beta = (C.c_double(1.0), C.c_double(0.0)) if ct == 1 else (C.c_float(1.0), C.c_float(0.0))
        size = C.c_size_t(0)
        if self.status == 0:
            self.status = R.cusparseSDDMM_bufferSize(self.h, NT, self.opB, C.byref(self.alpha), self.matA, self.matB, C.byref(self.beta),
                                                     self.matC, ct, 0, C.byref(size))
        self.buf = torch.empty(max(size.value, 16), dtype=torch.uint8, device=DEV)
        if self.status == 0:
            self.status = R.cusparseSDDMM_preprocess(self.h, NT, self.opB, C.byref(self.alpha), self.matA, self.matB, C.byref(self.beta),
                                                     self.matC, ct, 0, C.c_void_p(self.buf.data_ptr()))

    def __call__(self):
        st = self.R.cusparseSDDMM(self.h, NT, self.opB, C.byref(self.alpha), self.matA, self.matB, C.byref(self.beta), self.matC, self.ct, 0,
                                  C.c_void_p(self.buf.data_ptr()))
        assert st == 0, st

    def close(self):
        self.R.cusparseDestroySpMat(self.matC)
        self.api.cusparseDestroyDnMat(self.matA)
        self.api.cusparseDestroyDnMat(self.matB)
        self.api.cusparseDestroy(self.h)


def run_case(L, name, m, bs, k, dt, ctype, layout, off_np, col_np, batch=1, seed=1):
    n = m
    off = torch.tensor(off_np, device=DEV)
    col = torch.tensor(col_np, device=DEV)
    bnnz = int(col.numel())
    A, B = operands(m, n, k, dt, layout, seed, batch)
    ours_v = torch.zeros(batch * bnnz * bs * bs, dtype=ctype, device=DEV)
    closed_v = torch.zeros_like(ours_v)
    f64 = dt == torch.float64
    one, zero = (C.c_double(1.0), C.c_double(0.0)) if f64 else (C.c_float(1.0), C.c_float(0.0))
    sbk, sbj = (n, 1) if layout == "sample" else (1, k)
    stream = torch.cuda.current_stream().cuda_stream

    def ours():
        rc = L.b200sddmm_bsr(stream, VT[dt], VT[ctype], m, n, k, bs, bnnz, off.data_ptr(), col.data_ptr(), ours_v.data_ptr(), 0, 1,
                             C.addressof(one), C.addressof(zero), 0, A.data_ptr(), k, 1, B.data_ptr(), sbk, sbj, batch, 0, 0,
                             bnnz * bs * bs, m * k if batch > 1 else 0, n * k if batch > 1 else 0)
        assert rc == 0, rc
    ct = 1 if f64 else 0
    closed = Closed(m, n, k, bs, off, col, closed_v, A, B, layout, ct, batch)
    row = dict(case=name, m=m, bs=bs, k=k, type=f"{str(dt)[6:]}->{str(ctype)[6:]}", layout=layout, batch=batch, bnnz=bnnz,
               path="tensor" if L.b200sddmm_bsr_path(VT[dt], bs, A.data_ptr(), k, 1, B.data_ptr(), sbk, sbj, batch,
                                                     m * k if batch > 1 else 0, n * k if batch > 1 else 0) else "cuda-core")
    t_ours = timeit(ours)
    row["us_ours"] = t_ours * 1e6
    row["err_ours"] = reference_error(off, col, ours_v, A, B, bs, layout)
    if closed.status == 0:
        t_cl = timeit(closed)
        row["us_closed"] = t_cl * 1e6
        row["err_closed"] = reference_error(off, col, closed_v, A, B, bs, layout)
        row["speedup"] = t_cl / t_ours
    else:
        row["closed_status"] = closed.status
    closed.close()
    flops = 2.0 * bnnz * bs * bs * k * batch
    es = A.element_size()
    nbr = m // bs
    used_rows = int((np.diff(off_np) > 0).sum()) * bs
    used_cols = len(np.unique(col_np)) * bs
    bytes_ = (used_rows + used_cols) * k * es * batch + bnnz * bs * bs * ours_v.element_size() * batch + (nbr + 1 + bnnz) * 4
    t_flop, t_byte = flops / PEAK[dt], bytes_ / PEAK_BYTES
    row["tflops_ours"] = flops / t_ours / 1e12
    row["bound"] = "flops" if t_flop >= t_byte else "bytes"
    row["bound_us"] = max(t_flop, t_byte) * 1e6
    return row


def status_grid(L):
    """which combinations the closed library accepts: statuses of bufferSize + SDDMM over type x bs x op x order x batch layout"""
    R = _lib.real()
    api = cs.Api("cusparse")
    h = api.cusparseCreate()
    out = []
    m = n = 256
    k = 32
    buf = torch.empty(1 << 24, dtype=torch.uint8, device=DEV)

    def one(dt, ctype, compute, bs, opA, opB, oa, ob, oc, batch=1, share=(False, False, False, False, False)):
        nb = m // bs
        off = torch.arange(0, nb + 1, dtype=torch.int32, device=DEV)
        col = torch.arange(0, nb, dtype=torch.int32, device=DEV)
        A = torch.zeros(batch * m * k, dtype=dt, device=DEV)
        B = torch.zeros(batch * m * k, dtype=dt, device=DEV)
        V = torch.zeros(batch * nb * bs * bs, dtype=ctype, device=DEV)
        ar, ac = (m, k) if opA == NT else (k, m)
        br, bc = (k, n) if opB == NT else (n, k)
        mA = api.cusparseCreateDnMat(ar, ac, ac if oa == ROW else ar, A, oa)
        mB = api.cusparseCreateDnMat(br, bc, bc if ob == ROW else br, B, ob)
        d = C.c_void_p()
        st = R.cusparseCreateBsr(C.byref(d), C.c_int64(nb), C.c_int64(nb), C.c_int64(nb), C.c_int64(bs), C.c_int64(bs),
                                 C.c_void_p(off.data_ptr()), C.c_void_p(col.data_ptr()), C.c_void_p(V.data_ptr()), 2, 2, 0, VT[ctype], oc)
        sts = {"create": st}
        if st == 0:
            if batch > 1:
                if not share[2]:
                    api.cusparseDnMatSetStridedBatch(mA, batch, m * k)
                if not share[3]:
                    api.cusparseDnMatSetStridedBatch(mB, batch, m * k)
                sts["setStridedBatch"] = R.cusparseBsrSetStridedBatch(d, batch, C.c_int64(0 if share[0] else nb + 1), C.c_int64(0 if share[1] else nb),
                                                            C.c_int64(nb * bs * bs))
            al, be = (C.c_double(1), C.c_double(0)) if compute == 1 else (C.c_float(1), C.c_float(0))
            size = C.c_size_t(0)
            sts["bufferSize"] = R.cusparseSDDMM_bufferSize(h, opA, opB, C.byref(al), mA, mB, C.byref(be), d, compute, 0, C.byref(size))
            if sts["bufferSize"] == 0 and size.value <= buf.numel():
                sts["preprocess"] = R.cusparseSDDMM_preprocess(h, opA, opB, C.byref(al), mA, mB, C.byref(be), d, compute, 0,
                                                               C.c_void_p(buf.data_ptr()))
                sts["sddmm"] = R.cusparseSDDMM(h, opA, opB, C.byref(al), mA, mB, C.byref(be), d, compute, 0, C.c_void_p(buf.data_ptr()))
            torch.cuda.synchronize()
            R.cusparseDestroySpMat(d)
        api.cusparseDestroyDnMat(mA)
        api.cusparseDestroyDnMat(mB)
        return sts
    types = [(torch.float16, torch.float16, 0), (torch.float16, torch.float32, 0), (torch.bfloat16, torch.bfloat16, 0),
             (torch.bfloat16, torch.float32, 0), (torch.float32, torch.float32, 0), (torch.float64, torch.float64, 1),
             (torch.float16, torch.float16, 2), (torch.float32, torch.float32, 1)]
    for dt, ctype, compute in types:
        for bs in (1, 2, 4, 8, 16, 32, 64, 128):
            for opA in (NT, TR):
                for opB in (NT, TR):
                    for oc in (ROW, COL):
                        out.append(dict(type=f"{str(dt)[6:]}->{str(ctype)[6:]}/{compute}", bs=bs, opA=opA, opB=opB, orderC=oc,
                                        **one(dt, ctype, compute, bs, opA, opB, ROW, ROW, oc)))
                        print(json.dumps(out[-1]), flush=True)
    for dt, ctype, compute in types[:6]:
        for bs in (4, 16):
            for oa in (ROW, COL):
                for ob in (ROW, COL):
                    out.append(dict(type=f"{str(dt)[6:]}->{str(ctype)[6:]}/{compute}", bs=bs, orderA=oa, orderB=ob,
                                    **one(dt, ctype, compute, bs, NT, NT, oa, ob, ROW)))
                    print(json.dumps(out[-1]), flush=True)
    for dt, ctype, compute in types[:6]:
        for share in ((False,) * 5, (True, False, False, False, False), (True, True, False, False, False), (False, False, True, False, False),
                      (False, False, False, True, False), (True, True, True, False, False)):
            out.append(dict(type=f"{str(dt)[6:]}->{str(ctype)[6:]}/{compute}", bs=16, batch=4,
                            shared="".join(c for c, s in zip("ocAB", share) if s) or "-", **one(dt, ctype, compute, 16, NT, TR, ROW, ROW, ROW, 4, share)))
            print(json.dumps(out[-1]), flush=True)
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
        status_grid(L)
    seqs = [4096] if args.quick else args.seq
    # the sample itself: 8 x 8, bs 4, K 8, fp32, both layouts
    for layout in ("sample", "attention"):
        rows.append(run_case(L, "sample", 8, 4, 8, torch.float32, torch.float32, layout, np.array([0, 1, 2], np.int32),
                             np.array([0, 1], np.int32)))
        print(json.dumps(rows[-1]), flush=True)
    for seq in seqs:
        for kind in ("window", "rand10", "rand30"):
            for bs in (16, 32, 64, 128):
                off, col = pattern(kind, seq // bs, seed=bs)
                for k in (64, 128):
                    for tname, dt, ctype in TYPES:
                        for layout in ("sample", "attention"):
                            if args.quick and (k == 128 or kind == "rand30"):
                                continue
                            rows.append(run_case(L, kind, seq, bs, k, dt, ctype, layout, off, col))
                            print(json.dumps(rows[-1]), flush=True)
    # 16 heads sharing one pattern
    for tname, dt, ctype in ([] if args.no_heads else TYPES):
        for bs in (16, 64):
            off, col = pattern("window", 4096 // bs, seed=bs)
            for layout in ("sample", "attention"):
                rows.append(run_case(L, "window-16heads", 4096, bs, 64, dt, ctype, layout, off, col, batch=16))
                print(json.dumps(rows[-1]), flush=True)
    print(f"# {len(rows)} cases in {time.time() - t0:.0f} s on {name}", flush=True)
    if args.json:
        with open(args.json, "w") as f:
            json.dump(dict(card=name, rows=rows), f, indent=1)


if __name__ == "__main__":
    main()
