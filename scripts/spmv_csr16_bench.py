#!/usr/bin/env python
"""Half-precision CSR SpMV, ours (b200spmv_csr16 behind the shim's cusparseSpMV) against the closed library's cusparseSpMV on the same
buffers, in one process (DESIGN.md 3.19).

y = A . x with A a CSR matrix of fp16 / bf16 values, x of A's type, y of A's type or fp32, fp32 compute.  Matrices: R-MAT 1M and 10M
with 16 per row (workloads.rmat_csr, the bench's matrices), uniform 2M with 16 per row, the 5-point Poisson operator on an 8192^2 grid
(the cg sample's matrix) and the 7-point Laplacian on 256^3; values from workloads.py, cast to 16 bits.  Types: f16 -> f16,
f16 -> f32, bf16 -> bf16, bf16 -> f32.

Each side is timed with CUDA events after a warm-up (median of three windows), ours with the buffer cusparseSpMV_bufferSize asks for
(the split walk).  Where the shim's route forwards a shape, ours is timed on b200spmv_csr16 itself with the same buffer (`via`).
Reported per case: us for ours and for the closed library, the speed-up, effective GB/s on 4 (rows + 1) + 6 nnz + 2 cols + |y| bytes
(|y| twice when beta != 0; beta = 0 here) and its share of the H100 SXM data sheet's 3.35 TB/s, and each side's largest error
against fp64 relative to sum_k |a_rk| |x_k| over sampled rows (the longest row among them).  The card's name and power limit are read
in the same run.  --status records the closed library's statuses of bufferSize / preprocess / SpMV over A type x y type x compute
type x alg x opA.  --variants times further builds of libb200spmv.so (e.g. another chunk size) in the same process.
usage: python scripts/spmv_csr16_bench.py [--quick] [--status] [--only-status] [--matrices a,b] [--variants so,...] [--json out.json]"""
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

PEAK_BYTES = 3.35e12                    # H100 SXM data sheet, HBM3
DEV = torch.device("cuda:0")
NT, TR, CT = 0, 1, 2
F32, F64, F16, BF16 = 0, 1, 2, 14
VT = {torch.float32: F32, torch.float64: F64, torch.float16: F16, torch.bfloat16: BF16}
TYPES = [("f16-f16", torch.float16, torch.float16), ("f16-f32", torch.float16, torch.float32), ("bf16-bf16", torch.bfloat16, torch.bfloat16),
         ("bf16-f32", torch.bfloat16, torch.float32)]
MATRICES = ("rmat1m", "rmat10m", "uniform2m", "poisson8192", "laplace256")
ALGS = {"DEFAULT": 0, "COO_ALG1": 1, "CSR_ALG1": 2, "CSR_ALG2": 3}

# The shapes b200spmv_route sends to b200spmv_csr16 (DESIGN.md 3.19), as the predicate the CPU route test evaluates over (A / x type,
# y type, rows, cols, nnz), with opA = N, fp32 compute, alg DEFAULT / CSR_ALG1 / CSR_ALG2 and int32 indices.
# Measured on an H100 at 700 W (DESIGN.md 3.19): only R-MAT 10M into a 16-bit y ran faster than the closed library (1.18x); R-MAT 1M
# (0.60-0.67x), uniform 2M (0.95-0.96x), both stencils (0.45-0.63x) and every fp32 y were slower.  So the route takes a 16-bit y
# from 10M rows at the measured density of 16 entries per row, and forwards the rest.
NATIVE = "lambda vt, yt, rows, cols, nnz: yt == vt and rows >= 10 << 20 and 16 * rows <= nnz < 17 * rows"


def bytes_moved(rows, cols, nnz, y_bytes, beta_nonzero=False):
    return 4 * (rows + 1) + 6 * nnz + 2 * cols + rows * y_bytes * (2 if beta_nonzero else 1)


def card():
    import subprocess
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name(0)


def timeit(fn, budget=0.05):
    for _ in range(5):
        fn()
    torch.cuda.synchronize()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record(); fn(); e.record(); torch.cuda.synchronize()
    one = max(s.elapsed_time(e) / 1e3, 1e-6)
    reps = int(min(500, max(5, budget / one)))
    ts = []
    for _ in range(3):
        s.record()
        for _ in range(reps):
            fn()
        e.record()
        torch.cuda.synchronize()
        ts.append(s.elapsed_time(e) / 1e3 / reps)
    return float(np.median(ts))


def matrix(name, dev=DEV):
    """(rows, cols, off, col, fp32 values) on the device, base 0, sorted columns"""
    from cudalibrarysamples_b200 import workloads as W
    if name in ("rmat1m", "rmat10m"):
        rows = (1 << 20) if name == "rmat1m" else 10 * (1 << 20)
        off, col, val = W.rmat_csr(rows, avg_nnz=16, seed=42, val_seed=43, dtype=torch.float32)
    elif name == "uniform2m":
        rows = 2 << 20
        g = torch.Generator(device=dev).manual_seed(5)
        col = torch.randint(0, rows, (rows * 16,), device=dev, generator=g, dtype=torch.int32)
        col = col.view(rows, 16).sort(dim=1).values.reshape(-1).contiguous()
        off = torch.arange(0, rows * 16 + 1, 16, device=dev, dtype=torch.int32)
        val = torch.rand(rows * 16, device=dev, generator=g, dtype=torch.float32) * 2 - 1
    elif name == "poisson8192":
        off, col, val = W.stencil5_csr(8192)
        rows = 8192 * 8192
    elif name == "laplace256":
        off, col, val = W.laplace7_csr(256, dtype=torch.float32)
        rows = 256 ** 3
    else:
        raise ValueError(name)
    return rows, rows, off.int().contiguous(), col.int().contiguous(), val.float()


def sample_rows(off, nsample=64):
    lens = (off[1:] - off[:-1]).cpu().numpy()
    rows = np.random.default_rng(0).permutation(len(lens))[:nsample - 1]
    return np.unique(np.concatenate([rows, [int(np.argmax(lens))]]))


def reference_error(off, col, vals, x, y, rows):
    """largest |y_r - fp64| / sum_k |a_rk| |x_k| over the sampled rows (16-bit inputs taken as they are)"""
    offc = off.cpu().numpy()
    err = 0.0
    for r in rows:
        s, e = int(offc[r]), int(offc[r + 1])
        if s == e:
            continue
        a = vals[s:e].double()
        xx = x[col[s:e].long()].double()
        ref = float((a * xx).sum())
        bound = float((a.abs() * xx.abs()).sum())
        err = max(err, abs(float(y[r]) - ref) / max(bound, 1e-300))
    return err


def run_case(name, rows, cols, off, col, val32, dt, yt, seed=1, variants=()):
    L = _lib.shim()
    nnz = col.numel()
    vals = val32.to(dt)
    g = torch.Generator(device=DEV).manual_seed(seed)
    x = (torch.rand(cols, device=DEV, generator=g) * 2 - 1).to(dt)
    arrays = dict(off=off, col=col, val=vals)
    route = L.b200spmv_route(1, NT, 0, 2, 2, VT[dt], VT[dt], VT[yt], F32, rows, cols, nnz)
    row = dict(case=name, rows=rows, nnz=nnz, type=f"{str(dt)[6:]}->{str(yt)[6:]}", route=route,
               path=L.b200spmv_csr16_path(col.data_ptr(), vals.data_ptr()))
    sample = sample_rows(off)
    closed_y = torch.zeros(rows, dtype=yt, device=DEV)
    closed = cs.SpMVOperator(cs.Api("cusparse"), "csr", rows, cols, arrays, y_dtype=yt, compute_dtype=torch.float32)
    row["closed_buffer_mb"] = closed.buffer_bytes / 2 ** 20
    t_cl = timeit(closed.prebuilt(x, closed_y))
    row["us_closed"] = t_cl * 1e6
    row["err_closed"] = reference_error(off, col, vals, x, closed_y, sample)
    closed.close()
    ours_y = torch.zeros(rows, dtype=yt, device=DEV)
    api = cs.Api("b200")
    ours = cs.SpMVOperator(api, "csr", rows, cols, arrays, y_dtype=yt, compute_dtype=torch.float32)
    row["buffer_mb"] = ours.buffer_bytes / 2 ** 20
    if route == 3:
        row["via"] = "cusparseSpMV"
        api.reset_stats()
        t = timeit(ours.prebuilt(x, ours_y))
        st = api.stats()
        assert st["forwarded"] == 0 and st["native"] > 0, st
    else:
        row["via"] = "b200spmv_csr16"
        ws = ours.buffer
        one, zero = C.c_float(1.0), C.c_float(0.0)
        stream = torch.cuda.current_stream().cuda_stream

        def direct():
            assert L.b200spmv_csr16(stream, VT[dt], VT[yt], rows, cols, nnz, off.data_ptr(), col.data_ptr(), vals.data_ptr(), 0,
                                    C.addressof(one), C.addressof(zero), 0, x.data_ptr(), ours_y.data_ptr(), ws.data_ptr(),
                                    ours.buffer_bytes) == 0
        t = timeit(direct)
    ours.close()
    row["us_ours"] = t * 1e6
    row["speedup"] = t_cl / t
    row["err_ours"] = reference_error(off, col, vals, x, ours_y, sample)
    b = bytes_moved(rows, cols, nnz, ours_y.element_size())
    row["gbs"] = b / t / 1e9
    row["share_of_datasheet_3.35TBs"] = b / t / PEAK_BYTES
    row["bound_us"] = b / PEAK_BYTES * 1e6
    for path in variants:                   # the same call on another build of the library (same ABI)
        V = _lib.load(path)
        wsb = V.b200spmv_csr16_workspace_bytes(rows, nnz)
        ws = torch.empty(max(wsb, 16), dtype=torch.uint8, device=DEV)
        vy = torch.zeros_like(ours_y)
        one, zero = C.c_float(1.0), C.c_float(0.0)
        stream = torch.cuda.current_stream().cuda_stream

        def var(V=V, ws=ws, wsb=wsb, vy=vy):
            assert V.b200spmv_csr16(stream, VT[dt], VT[yt], rows, cols, nnz, off.data_ptr(), col.data_ptr(), vals.data_ptr(), 0,
                                    C.addressof(one), C.addressof(zero), 0, x.data_ptr(), vy.data_ptr(), ws.data_ptr(), wsb) == 0
        row[f"us_{os.path.basename(path)}"] = timeit(var) * 1e6
    return row


def status_grid():
    """which combinations the closed library accepts for a 16-bit CSR A: statuses of bufferSize / preprocess / SpMV over A type x
    y type x compute type x alg x opA, at 256 x 256 with 4 per row"""
    R = _lib.real()
    api = cs.Api("cusparse")
    h = api.cusparseCreate()
    out = []
    m = 256
    buf = torch.empty(1 << 24, dtype=torch.uint8, device=DEV)
    off = torch.arange(0, 4 * m + 1, 4, dtype=torch.int32, device=DEV)
    col = ((torch.arange(4 * m, dtype=torch.int32, device=DEV) * 7) % m).view(m, 4).sort(dim=1).values.reshape(-1).contiguous()

    def one(at, xt, yt, compute, opA, alg):
        vals = torch.zeros(4 * m, dtype=at, device=DEV)
        x = torch.zeros(m, dtype=xt, device=DEV)
        y = torch.zeros(m, dtype=yt, device=DEV)
        vx, vy = api.cusparseCreateDnVec(m, x), api.cusparseCreateDnVec(m, y)
        d = C.c_void_p()
        st = R.cusparseCreateCsr(C.byref(d), C.c_int64(m), C.c_int64(m), C.c_int64(4 * m), C.c_void_p(off.data_ptr()),
                                 C.c_void_p(col.data_ptr()), C.c_void_p(vals.data_ptr()), 2, 2, 0, VT[at])
        sts = {"create": st}
        if st == 0:
            if compute == F64:
                al, be = C.c_double(1), C.c_double(0)
            elif compute in (F16, BF16):
                al, be = C.c_uint16(0x3C00 if compute == F16 else 0x3F80), C.c_uint16(0)
            else:
                al, be = C.c_float(1), C.c_float(0)
            size = C.c_size_t(0)
            sts["bufferSize"] = R.cusparseSpMV_bufferSize(h, opA, C.byref(al), d, vx, C.byref(be), vy, compute, alg, C.byref(size))
            if sts["bufferSize"] == 0 and size.value <= buf.numel():
                sts["preprocess"] = R.cusparseSpMV_preprocess(h, opA, C.byref(al), d, vx, C.byref(be), vy, compute, alg,
                                                              C.c_void_p(buf.data_ptr()))
                sts["spmv"] = R.cusparseSpMV(h, opA, C.byref(al), d, vx, C.byref(be), vy, compute, alg, C.c_void_p(buf.data_ptr()))
            torch.cuda.synchronize()
            R.cusparseDestroySpMat(d)
        api.cusparseDestroyDnVec(vx)
        api.cusparseDestroyDnVec(vy)
        return sts

    f16, bf16, f32 = torch.float16, torch.bfloat16, torch.float32
    combos = [(f16, f16, f16, F32), (f16, f16, f32, F32), (bf16, bf16, bf16, F32), (bf16, bf16, f32, F32),   # the served pairs
              (f16, f16, f16, F16), (bf16, bf16, bf16, BF16),                                                 # 16-bit compute
              (f16, f16, bf16, F32), (bf16, bf16, f16, F32), (f16, bf16, f32, F32), (f16, f32, f32, F32)]     # mixed
    for at, xt, yt, compute in combos:
        t = f"A {str(at)[6:]} x {str(xt)[6:]} y {str(yt)[6:]} compute {compute}"
        for opA in (NT, TR, CT):
            for aname, alg in ALGS.items():
                kw = dict(type=t, opA=opA, alg=aname)
                kw.update(one(at, xt, yt, compute, opA, alg))
                out.append(kw)
                print(json.dumps(kw), flush=True)
    api.cusparseDestroy(h)
    return out


def quick_rehearsal():
    """the host logic at a tiny size on the CPU: byte model, reference error, the NATIVE predicate; timing needs a GPU"""
    off = torch.tensor([0, 2, 2, 5], dtype=torch.int32)
    col = torch.tensor([0, 2, 1, 2, 3], dtype=torch.int32)
    vals = torch.tensor([1, -2, 3, 0.5, 1], dtype=torch.float16)
    x = torch.tensor([1, 2, -1, 4], dtype=torch.float16)
    y = torch.tensor([3, 0, 9.5], dtype=torch.float32)
    assert reference_error(off, col, vals, x, y, sample_rows(off)) == 0.0
    assert bytes_moved(3, 4, 5, 4) == 4 * 4 + 30 + 8 + 12
    assert eval(NATIVE)(F16, F32, 1 << 20, 1 << 20, 16 << 20) in (True, False)
    print("# quick: host logic OK at 3 x 4", flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--quick", action="store_true", help="CPU rehearsal of the host logic, then R-MAT 1M only")
    ap.add_argument("--status", action="store_true", help="also print the closed library's status grid")
    ap.add_argument("--only-status", action="store_true")
    ap.add_argument("--matrices", default=",".join(MATRICES))
    ap.add_argument("--types", default=",".join(t[0] for t in TYPES))
    ap.add_argument("--variants", default="", help="comma-separated further builds of libb200spmv.so to time in the same process")
    ap.add_argument("--json")
    args = ap.parse_args()
    if args.quick:
        quick_rehearsal()
    if not torch.cuda.is_available():
        raise SystemExit("no GPU: the timing run needs one")
    name = card()
    print(f"# card: {name}", flush=True)
    rows_out, status = [], []
    t0 = time.time()
    if args.status or args.only_status:
        status = status_grid()
    variants = [v for v in args.variants.split(",") if v]
    mats = [] if args.only_status else ["rmat1m"] if args.quick else args.matrices.split(",")
    for mname in mats:
        rows, cols, off, col, val = matrix(mname)
        for tname, dt, yt in TYPES:
            if tname in args.types.split(","):
                rows_out.append(run_case(mname, rows, cols, off, col, val, dt, yt, variants=variants))
                print(json.dumps(rows_out[-1]), flush=True)
        del off, col, val
        torch.cuda.empty_cache()
    print(f"# {len(rows_out)} cases in {time.time() - t0:.0f} s on {name}", flush=True)
    if args.json:
        with open(args.json, "w") as f:
            json.dump(dict(card=name, rows=rows_out, status=status), f, indent=1)


if __name__ == "__main__":
    main()
