#!/usr/bin/env python
"""Half-precision CSR SpMM, ours (b200spmm_csr16) against the closed library's cusparseSpMM on the same buffers, in one process
(DESIGN.md 3.18).

C = A . B with A a CSR matrix of fp16 / bf16 values and B dense: graph aggregation (A the adjacency of a power-law graph) and
pruned-weight inference.  Matrices: R-MAT 1M x 1M with 16 per row (workloads.rmat_csr, the project's headline matrix), R-MAT 2M x 2M
with 32 per row, and uniform 2M x 2M with 32 per row (the shape of BASELINE config 5); values in [-1, 1) cast to 16 bits.  N (columns
of B and C) 32, 64, 128, 256.  Types: f16 -> f16, f16 -> f32, bf16 -> bf16, bf16 -> f32, fp32 compute.  Orders: B and C both
row-major, and both column-major (opB = N).

Each call is timed with CUDA events after a warm-up (median of three windows).  Reported per case: us for ours (with the workspace the
shim passes: the split walk, and the row-major copy of a column-major B) and for the closed library, the speed-up, effective GB/s
on two byte models -- `gbs` on A (values, columns, offsets) + B once + C, the traffic no implementation avoids, and `gather_gbs` on
the gathered volume nnz * N * 2 bytes, which L2 serves in part -- and each side's largest error against fp64 relative to
sum_k |a_ik| |b_kj| over sampled rows (the longest row among them).  The card's name and power limit are read in the same run.
--status records the closed library's statuses of bufferSize / preprocess / SpMM over type x C type x opB x order x alg.
usage: python scripts/spmm_csr16_bench.py [--quick] [--status] [--only-status] [--json out.json]"""
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
from cudalibrarysamples_b200 import workloads as W  # noqa: E402
from scripts.sddmm_bsr_bench import PEAK_BYTES, card, timeit  # noqa: E402

DEV = torch.device("cuda:0")
ROW, COL = cs.CUSPARSE_ORDER_ROW, cs.CUSPARSE_ORDER_COL
NT, TR = cs.CUSPARSE_OPERATION_NON_TRANSPOSE, cs.CUSPARSE_OPERATION_TRANSPOSE
VT = {torch.float32: 0, torch.float64: 1, torch.float16: 2, torch.bfloat16: 14}
TYPES = [("f16-f16", torch.float16, torch.float16), ("f16-f32", torch.float16, torch.float32), ("bf16-bf16", torch.bfloat16, torch.bfloat16),
         ("bf16-f32", torch.bfloat16, torch.float32)]
MATRICES = ("rmat1m", "rmat2m", "uniform2m")

# The classes b200spmm_csr16_route runs natively (DESIGN.md 3.18), as the predicate the CPU route test evaluates over (A / B type,
# C type, N, rows, nnz, order of B and C) with opB = N and B and C in one order (COL = 1): every case measured in a class ran at
# least at parity.  Row-major N = 128 lost on R-MAT 1M (0.83x - 0.92x) and, into an fp32 C, on R-MAT 2M (0.95x - 0.97x).
NATIVE = ("lambda vt, cvt, n, m, nnz, order: m >= 1 << 20 and nnz >= 16 * m and 32 <= n <= 256 and (order == 1 or n <= 64 "
          "or n == 256 or (n == 128 and cvt == vt and m >= 2 << 20 and nnz >= 32 * m))")


def matrix(name):
    """(rows, off, col, fp32 values) on the device, base 0, sorted columns"""
    if name == "rmat1m":
        rows = 1 << 20
        off, col, val = W.rmat_csr(rows, avg_nnz=16, seed=42, val_seed=43, dtype=torch.float32)
    elif name == "rmat2m":
        rows = 2 << 20
        off, col, val = W.rmat_csr(rows, avg_nnz=32, seed=44, val_seed=45, dtype=torch.float32)
    else:
        rows = 2 << 20
        g = torch.Generator(device=DEV).manual_seed(5)
        col = torch.randint(0, rows, (rows * 32,), device=DEV, generator=g, dtype=torch.int32)
        col = col.view(rows, 32).sort(dim=1).values.reshape(-1).contiguous()
        off = torch.arange(0, rows * 32 + 1, 32, device=DEV, dtype=torch.int32)
        val = torch.rand(rows * 32, device=DEV, generator=g, dtype=torch.float32) * 2 - 1
    return rows, off.int().contiguous(), col.int().contiguous(), val.float()


class Closed:
    """the closed library's cusparseSpMM on a 16-bit CSR A, descriptors built once"""

    def __init__(self, m, k, n, off, col, vals, Bt, Cb, order, opB=NT, alg=0):
        self.api = cs.Api("cusparse")
        R = self.R = self.api.real
        self.h = self.api.cusparseCreate()
        br, bc = (k, n) if opB == NT else (n, k)
        self.matB = self.api.cusparseCreateDnMat(br, bc, bc if order == ROW else br, Bt, order)
        self.matC = self.api.cusparseCreateDnMat(m, n, n if order == ROW else m, Cb, order)
        d = C.c_void_p()
        assert R.cusparseCreateCsr(C.byref(d), C.c_int64(m), C.c_int64(k), C.c_int64(col.numel()), C.c_void_p(off.data_ptr()),
                                   C.c_void_p(col.data_ptr()), C.c_void_p(vals.data_ptr()), 2, 2, 0, VT[vals.dtype]) == 0
        self.matA = d
        self.opB, self.alg = opB, alg
        self.alpha, self.beta = C.c_float(1.0), C.c_float(0.0)
        size = C.c_size_t(0)
        self.status = R.cusparseSpMM_bufferSize(self.h, NT, opB, C.byref(self.alpha), self.matA, self.matB, C.byref(self.beta), self.matC,
                                                0, alg, C.byref(size))
        self.size = size.value
        self.buf = torch.empty(max(size.value, 16), dtype=torch.uint8, device=DEV)
        if self.status == 0:
            self.status = R.cusparseSpMM_preprocess(self.h, NT, opB, C.byref(self.alpha), self.matA, self.matB, C.byref(self.beta),
                                                    self.matC, 0, alg, C.c_void_p(self.buf.data_ptr()))

    def __call__(self):
        st = self.R.cusparseSpMM(self.h, NT, self.opB, C.byref(self.alpha), self.matA, self.matB, C.byref(self.beta), self.matC, 0,
                                 self.alg, C.c_void_p(self.buf.data_ptr()))
        assert st == 0, st

    def close(self):
        self.R.cusparseDestroySpMat(self.matA)
        self.api.cusparseDestroyDnMat(self.matB)
        self.api.cusparseDestroyDnMat(self.matC)
        self.api.cusparseDestroy(self.h)


def sample_rows(off, nsample=48):
    lens = (off[1:] - off[:-1]).cpu().numpy()
    rows = np.random.default_rng(0).permutation(len(lens))[:nsample - 1]
    return np.unique(np.concatenate([rows, [int(np.argmax(lens))]]))


def reference_error(off, col, vals, Bd, got, m, n, order, rows):
    """largest |c - fp64| / sum_k |a_ik| |b_kj| over the sampled rows; Bd is op(B) as fp64 (k x n)"""
    Cd = got[:m * n].view(m, n) if order == ROW else got[:m * n].view(n, m).t()
    offc = off.cpu().numpy()
    err = 0.0
    for r in rows:
        s, e = int(offc[r]), int(offc[r + 1])
        if s == e:
            continue
        a = vals[s:e].double()
        bb = Bd[col[s:e].long()]
        ref = a @ bb
        bound = a.abs() @ bb.abs()
        d = (Cd[r].double() - ref).abs() / bound.clamp(min=1e-300)
        err = max(err, float(d.max()))
    return err


def run_case(L, name, m, off, col, val32, n, dt, ctype, order, seed=1, split=True):
    k = m
    nnz = col.numel()
    vals = val32.to(dt)
    g = torch.Generator(device=DEV).manual_seed(seed)
    Bop = (torch.rand(k, n, device=DEV, generator=g) * 2 - 1).to(dt)            # op(B), k x n
    Bs = Bop.contiguous() if order == ROW else Bop.t().contiguous()              # stored in the order
    ours_c = torch.zeros(m * n, dtype=ctype, device=DEV)
    closed_c = torch.zeros_like(ours_c)
    one, zero = C.c_float(1.0), C.c_float(0.0)
    sbk, sbj = (n, 1) if order == ROW else (1, k)
    ldc = n if order == ROW else m
    wsb = L.b200spmm_csr16_workspace_bytes(k, n, nnz, sbk, sbj) if split else 0
    ws = torch.empty(max(wsb, 16), dtype=torch.uint8, device=DEV)
    stream = torch.cuda.current_stream().cuda_stream

    def ours():
        rc = L.b200spmm_csr16(stream, VT[dt], VT[ctype], m, k, n, nnz, off.data_ptr(), col.data_ptr(), vals.data_ptr(), 0,
                              C.addressof(one), C.addressof(zero), 0, Bs.data_ptr(), sbk, sbj, ours_c.data_ptr(), ldc,
                              1 if order == ROW else 0, ws.data_ptr() if split else None, wsb)
        assert rc == 0, rc
    closed = Closed(m, k, n, off, col, vals, Bs, closed_c, order)
    path = L.b200spmm_csr16_path(n, Bs.data_ptr(), sbk, sbj) if order == ROW else L.b200spmm_csr16_path(n, ws.data_ptr(), n, 1)
    row = dict(case=name, m=m, nnz=nnz, n=n, type=f"{str(dt)[6:]}->{str(ctype)[6:]}", order="row" if order == ROW else "col",
               path=path, ws_mb=wsb / 2 ** 20, closed_ws_mb=closed.size / 2 ** 20)
    t_ours = timeit(ours)
    row["us_ours"] = t_ours * 1e6
    rows = sample_rows(off)
    Bd = Bop.double()
    row["err_ours"] = reference_error(off, col, vals, Bd, ours_c, m, n, order, rows)
    if closed.status == 0:
        t_cl = timeit(closed)
        row["us_closed"] = t_cl * 1e6
        row["err_closed"] = reference_error(off, col, vals, Bd, closed_c, m, n, order, rows)
        row["speedup"] = t_cl / t_ours
    else:
        row["closed_status"] = closed.status
    closed.close()
    used = int(torch.unique(col).numel())
    bytes_min = nnz * (2 + 4) + (m + 1) * 4 + used * n * 2 + m * n * ours_c.element_size()
    row["gbs"] = bytes_min / t_ours / 1e9
    row["gather_gbs"] = nnz * n * 2 / t_ours / 1e9
    row["bound_us"] = bytes_min / PEAK_BYTES * 1e6
    del Bop, Bs, ours_c, closed_c, ws
    return row


def status_grid():
    """which combinations the closed library accepts for a 16-bit CSR A: statuses of bufferSize / preprocess / SpMM over type x C
    type x compute x opB x order of B and C x alg"""
    R = _lib.real()
    api = cs.Api("cusparse")
    h = api.cusparseCreate()
    out = []
    m, n = 256, 64
    buf = torch.empty(1 << 24, dtype=torch.uint8, device=DEV)
    off = torch.arange(0, 4 * m + 1, 4, dtype=torch.int32, device=DEV)
    col = (torch.arange(4 * m, dtype=torch.int32, device=DEV) * 7) % m
    col = col.view(m, 4).sort(dim=1).values.reshape(-1).contiguous()

    def one(dt, ctype, compute, opB, ob, oc, alg):
        vals = torch.zeros(4 * m, dtype=dt, device=DEV)
        B = torch.zeros(m * n, dtype=dt, device=DEV)
        Cm = torch.zeros(m * n, dtype=ctype, device=DEV)
        br, bc = (m, n) if opB == NT else (n, m)
        mB = api.cusparseCreateDnMat(br, bc, bc if ob == ROW else br, B, ob)
        mC = api.cusparseCreateDnMat(m, n, n if oc == ROW else m, Cm, oc)
        d = C.c_void_p()
        st = R.cusparseCreateCsr(C.byref(d), C.c_int64(m), C.c_int64(m), C.c_int64(4 * m), C.c_void_p(off.data_ptr()),
                                 C.c_void_p(col.data_ptr()), C.c_void_p(vals.data_ptr()), 2, 2, 0, VT[dt])
        sts = {"create": st}
        if st == 0:
            al, be = (C.c_double(1), C.c_double(0)) if compute == 1 else (C.c_float(1), C.c_float(0))
            if compute == 2:
                al, be = C.c_uint16(0x3C00), C.c_uint16(0)
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

    types = [(torch.float16, torch.float16, 0), (torch.float16, torch.float32, 0), (torch.bfloat16, torch.bfloat16, 0),
             (torch.bfloat16, torch.float32, 0), (torch.float16, torch.float16, 2), (torch.bfloat16, torch.float16, 0),
             (torch.float16, torch.bfloat16, 0)]
    algs = {"DEFAULT": 0, "CSR_ALG1": 4, "CSR_ALG2": 6, "CSR_ALG3": 12}
    for dt, ctype, compute in types:
        t = f"{str(dt)[6:]}->{str(ctype)[6:]}/{compute}"
        for opB in (NT, TR):
            for ob in (ROW, COL):
                for oc in (ROW, COL):
                    for aname, alg in algs.items():
                        kw = dict(type=t, opB=opB, orderB="row" if ob == ROW else "col", orderC="row" if oc == ROW else "col", alg=aname)
                        kw.update(one(dt, ctype, compute, opB, ob, oc, alg))
                        out.append(kw)
                        print(json.dumps(kw), flush=True)
    api.cusparseDestroy(h)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--quick", action="store_true", help="R-MAT 1M, N 64 / 128, row-major only")
    ap.add_argument("--status", action="store_true", help="also print the closed library's status grid")
    ap.add_argument("--only-status", action="store_true")
    ap.add_argument("--json")
    args = ap.parse_args()
    L = _lib.shim()
    name = card()
    print(f"# card: {name}", flush=True)
    rows, status = [], []
    t0 = time.time()
    if args.status or args.only_status:
        status = status_grid()
    for mname in ([] if args.only_status else ["rmat1m"] if args.quick else MATRICES):
        m, off, col, val = matrix(mname)
        for n in ((64, 128) if args.quick else (32, 64, 128, 256)):
            for tname, dt, ctype in TYPES:
                for order in ((ROW,) if args.quick else (ROW, COL)):
                    rows.append(run_case(L, mname, m, off, col, val, n, dt, ctype, order))
                    print(json.dumps(rows[-1]), flush=True)
        del off, col, val
        torch.cuda.empty_cache()
    print(f"# {len(rows)} cases in {time.time() - t0:.0f} s on {name}", flush=True)
    if args.json:
        with open(args.json, "w") as f:
            json.dump(dict(card=name, rows=rows, status=status), f, indent=1)


if __name__ == "__main__":
    main()
