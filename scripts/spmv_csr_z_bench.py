#!/usr/bin/env python
"""Double-complex CSR SpMV, ours (b200spmv_csr_z behind the shim's cusparseSpMV) against the closed library's cusparseSpMV on the same
buffers, in one process (DESIGN.md 3.21).

y = alpha * op(A) * x + beta * y with A a CSR matrix of CUDA_C_64F values, x, y and compute CUDA_C_64F, opA N / T / C.  Matrices:
R-MAT 1M and 10M with 16 per row (workloads.rmat_csr, the bench's matrices), uniform 2M with 16 per row, the 5-point Poisson operator
on an 8192^2 grid (the cg sample's matrix) and the 7-point Laplacian on 256^3.  A's real parts are the workload's values, its imaginary
parts and x are drawn from the same seeds.  Each case runs with beta = 0 and with beta != 0.

The two sides are timed alternately with CUDA events after a warm-up (median of three windows each), ours with the buffer our
kernel asks for (the split walk).  Where the shim's route forwards a case, ours is timed on b200spmv_csr_z itself (`via`).  Reported
per case: us for ours and for the closed library, the speed-up, effective GB/s on 4 (rows + 1) + 20 nnz + 16 |x| + 16 |y| bytes (|y|
twice when beta != 0) and its share of the H100 SXM data sheet's 3.35 TB/s, and each side's largest error against an fp64 reference
relative to sum |alpha| |a| |x| + |beta| |y0| per entry of y.  The card's name and power limit are read in the same run.  --status
records the closed library's statuses of bufferSize / preprocess / SpMV over value type x opA x alg.  --variants times further builds
of libb200spmv.so (e.g. another chunk size) for opA = N in the same process.
usage: python scripts/spmv_csr_z_bench.py [--quick] [--status] [--only-status] [--matrices a,b] [--variants so,...] [--json out.json]"""
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
OPS = {"N": NT, "T": TR, "C": CT}
R32, R64, C32, C64 = 0, 1, 4, 5
MATRICES = ("rmat1m", "rmat10m", "uniform2m", "poisson8192", "laplace256")
ALGS = {"DEFAULT": 0, "COO_ALG1": 1, "CSR_ALG1": 2, "CSR_ALG2": 3}
ALPHA, BETA = 0.75 + 0.5j, 0.5 - 0.25j

# The cases b200spmv_route sends to b200spmv_csr_z (DESIGN.md 3.21), as the predicate the CPU route test evaluates over (opA, rows,
# cols, nnz), with A, x, y and compute CUDA_C_64F, alg DEFAULT / CSR_ALG1 / CSR_ALG2 and int32 indices.
# Measured on an H100 at 700 W (DESIGN.md 3.21): opA = N 0.40-0.99x of the closed library, T / C 0.63-0.996x, on every matrix here.
# No case reached parity, so the route takes none.
NATIVE = "lambda op, rows, cols, nnz: False"


def bytes_moved(rows, cols, nnz, op, beta_nonzero=False):
    nx, ny = (cols, rows) if op == NT else (rows, cols)
    return 4 * (rows + 1) + 20 * nnz + 16 * nx + 16 * ny * (2 if beta_nonzero else 1)


def card():
    import subprocess
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name(0)


def timeit_pair(fa, fb, budget=0.05, rounds=3):
    """median seconds per call of fa and of fb, timed in alternating windows after a warm-up of both"""
    for _ in range(5):
        fa()
        fb()
    torch.cuda.synchronize()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record(); fa(); e.record(); torch.cuda.synchronize()
    one = max(s.elapsed_time(e) / 1e3, 1e-6)
    reps = int(min(500, max(5, budget / one)))
    ta, tb = [], []
    for _ in range(rounds):
        for fn, out in ((fa, ta), (fb, tb)):
            s.record()
            for _ in range(reps):
                fn()
            e.record()
            torch.cuda.synchronize()
            out.append(s.elapsed_time(e) / 1e3 / reps)
    return float(np.median(ta)), float(np.median(tb))


def matrix(name, dev=DEV):
    """(rows, cols, off, col, complex128 values) on the device, base 0, sorted columns"""
    from cudalibrarysamples_b200 import workloads as W
    if name in ("rmat1m", "rmat10m"):
        rows = (1 << 20) if name == "rmat1m" else 10 * (1 << 20)
        off, col, val = W.rmat_csr(rows, avg_nnz=16, seed=42, val_seed=43, dtype=torch.float64)
    elif name == "uniform2m":
        rows = 2 << 20
        g = torch.Generator(device=dev).manual_seed(5)
        col = torch.randint(0, rows, (rows * 16,), device=dev, generator=g, dtype=torch.int32)
        col = col.view(rows, 16).sort(dim=1).values.reshape(-1).contiguous()
        off = torch.arange(0, rows * 16 + 1, 16, device=dev, dtype=torch.int32)
        val = torch.rand(rows * 16, device=dev, generator=g, dtype=torch.float64) * 2 - 1
    elif name == "poisson8192":
        off, col, val = W.stencil5_csr(8192)
        rows = 8192 * 8192
    elif name == "laplace256":
        off, col, val = W.laplace7_csr(256, dtype=torch.float64)
        rows = 256 ** 3
    else:
        raise ValueError(name)
    g = torch.Generator(device=dev).manual_seed(7)
    imag = torch.rand(col.numel(), device=dev, generator=g, dtype=torch.float64) * 2 - 1
    vals = torch.complex(val.double(), imag)
    del val, imag
    return rows, rows, off.int().contiguous(), col.int().contiguous(), vals


def reference(off, col, vals, x, op, y0, alpha, beta):
    """fp64 alpha * op(A) x + beta * y0 and the bound sum |alpha| |a| |x| + |beta| |y0| per entry of y, by index_add on the device"""
    rows = off.numel() - 1
    lens = (off[1:] - off[:-1]).long()
    row = torch.repeat_interleave(torch.arange(rows, device=DEV), lens)
    colL = col.long()
    if op == NT:
        src, dst, n = colL, row, rows
        v = vals
    else:
        src, dst, n = row, colL, y0.numel()
        v = vals.conj() if op == CT else vals
    ref = torch.zeros(n, dtype=torch.complex128, device=DEV)
    bound = torch.zeros(n, dtype=torch.float64, device=DEV)
    step = 1 << 26
    for i in range(0, v.numel(), step):
        sl = slice(i, i + step)
        p = v[sl] * x[src[sl]]
        ref.index_add_(0, dst[sl], p)
        bound.index_add_(0, dst[sl], p.abs())
    ref = alpha * ref
    bound = abs(alpha) * bound
    if beta != 0:
        ref = ref + beta * y0
        bound = bound + abs(beta) * y0.abs()
    return ref, bound


def rel_err(y, ref, bound):
    return float(((y - ref).abs() / (bound + 1e-300)).max())


def run_case(name, rows, cols, off, col, vals, op, beta, seed=1, variants=()):
    L = _lib.shim()
    nnz = col.numel()
    nx, ny = (cols, rows) if op == NT else (rows, cols)
    g = torch.Generator(device=DEV).manual_seed(seed)
    x = torch.complex(torch.rand(nx, device=DEV, generator=g, dtype=torch.float64) * 2 - 1,
                      torch.rand(nx, device=DEV, generator=g, dtype=torch.float64) * 2 - 1)
    y0 = torch.complex(torch.rand(ny, device=DEV, generator=g, dtype=torch.float64) * 2 - 1,
                       torch.rand(ny, device=DEV, generator=g, dtype=torch.float64) * 2 - 1)
    arrays = dict(off=off, col=col, val=vals)
    route = L.b200spmv_route(1, op, 0, 2, 2, C64, C64, C64, C64, rows, cols, nnz)
    opname = {NT: "N", TR: "T", CT: "C"}[op]
    row = dict(case=name, rows=rows, nnz=nnz, op=opname, beta=str(beta), route=route)
    ref, bound = reference(off, col, vals, x, op, y0, ALPHA, beta)
    closed_y, ours_y = y0.clone(), y0.clone()
    closed = cs.SpMVOperator(cs.Api("cusparse"), "csr", rows, cols, arrays, op=op)
    row["closed_buffer_mb"] = closed.buffer_bytes / 2 ** 20
    closed_call = closed.prebuilt(x, closed_y, ALPHA, beta)
    api = cs.Api("b200")
    ours = cs.SpMVOperator(api, "csr", rows, cols, arrays, op=op)
    one_a, one_b = cs.CDoubleComplex(ALPHA), cs.CDoubleComplex(beta)
    stream = torch.cuda.current_stream().cuda_stream
    wsb = L.b200spmv_csr_z_workspace_bytes(rows, nnz) if op == NT else 0
    ws = torch.empty(max(wsb, 16), dtype=torch.uint8, device=DEV)
    if route == 4:
        row["via"] = "cusparseSpMV"
        ours_call = ours.prebuilt(x, ours_y, ALPHA, beta)
    else:
        row["via"] = "b200spmv_csr_z"

        def ours_call():
            assert L.b200spmv_csr_z(stream, op, rows, cols, nnz, off.data_ptr(), col.data_ptr(), vals.data_ptr(), 0,
                                    C.addressof(one_a), C.addressof(one_b), 0, x.data_ptr(), ours_y.data_ptr(), ws.data_ptr(), wsb) == 0
    # one call each from y0 for the error, then the timing (beta != 0 keeps updating y; |beta| < 1 keeps it bounded)
    closed_call()
    ours_call()
    torch.cuda.synchronize()
    row["err_closed"] = rel_err(closed_y, ref, bound)
    row["err_ours"] = rel_err(ours_y, ref, bound)
    if route == 4:
        api.reset_stats()
    t_cl, t = timeit_pair(closed_call, ours_call)
    if route == 4:
        st = api.stats()
        assert st["forwarded"] == 0 and st["native"] > 0, st
    closed.close()
    ours.close()
    row["us_closed"] = t_cl * 1e6
    row["us_ours"] = t * 1e6
    row["speedup"] = t_cl / t
    b = bytes_moved(rows, cols, nnz, op, beta != 0)
    row["gbs"] = b / t / 1e9
    row["share_of_datasheet_3.35TBs"] = b / t / PEAK_BYTES
    row["bound_us"] = b / PEAK_BYTES * 1e6
    for path in (variants if op == NT else ()):     # the same call on another build of the library (same ABI)
        V = _lib.load(path)
        vwsb = V.b200spmv_csr_z_workspace_bytes(rows, nnz)
        vws = torch.empty(max(vwsb, 16), dtype=torch.uint8, device=DEV)
        vy = y0.clone()

        def var(V=V, vws=vws, vwsb=vwsb, vy=vy):
            assert V.b200spmv_csr_z(stream, op, rows, cols, nnz, off.data_ptr(), col.data_ptr(), vals.data_ptr(), 0,
                                    C.addressof(one_a), C.addressof(one_b), 0, x.data_ptr(), vy.data_ptr(), vws.data_ptr(), vwsb) == 0
        t_base, t_var = timeit_pair(ours_call, var)
        row[f"us_{os.path.basename(path)}"] = t_var * 1e6
        row[f"us_default_vs_{os.path.basename(path)}"] = t_base * 1e6
    return row


def status_grid():
    """which combinations the closed library accepts for a complex CSR A: statuses of bufferSize / preprocess / SpMV over A / x / y /
    compute type x alg x opA, at 256 x 256 with 4 per row"""
    R = _lib.real()
    api = cs.Api("cusparse")
    h = api.cusparseCreate()
    out = []
    m = 256
    buf = torch.empty(1 << 24, dtype=torch.uint8, device=DEV)
    off = torch.arange(0, 4 * m + 1, 4, dtype=torch.int32, device=DEV)
    col = ((torch.arange(4 * m, dtype=torch.int32, device=DEV) * 7) % m).view(m, 4).sort(dim=1).values.reshape(-1).contiguous()
    tdt = {R32: torch.float32, R64: torch.float64, C32: torch.complex64, C64: torch.complex128}

    def vec(n, t):
        v = torch.zeros(n, dtype=tdt[t], device=DEV)
        d = C.c_void_p()
        assert R.cusparseCreateDnVec(C.byref(d), C.c_int64(n), C.c_void_p(v.data_ptr()), t) == 0
        return d, v

    def one(at, xt, yt, compute, opA, alg):
        vals = torch.zeros(4 * m, dtype=tdt[at], device=DEV)
        (vx, kx), (vy, ky) = vec(m, xt), vec(m, yt)
        d = C.c_void_p()
        st = R.cusparseCreateCsr(C.byref(d), C.c_int64(m), C.c_int64(m), C.c_int64(4 * m), C.c_void_p(off.data_ptr()),
                                 C.c_void_p(col.data_ptr()), C.c_void_p(vals.data_ptr()), 2, 2, 0, at)
        sts = {"create": st}
        if st == 0:
            if compute == C64:
                al, be = cs.CDoubleComplex(1), cs.CDoubleComplex(0)
            elif compute == C32:
                al, be = (C.c_float * 2)(1, 0), (C.c_float * 2)(0, 0)
            elif compute == R64:
                al, be = C.c_double(1), C.c_double(0)
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
        R.cusparseDestroyDnVec(vx)
        R.cusparseDestroyDnVec(vy)
        return sts

    combos = [(C64, C64, C64, C64), (C32, C32, C32, C32), (C32, C64, C64, C64), (R64, C64, C64, C64), (C32, C32, C32, C64),
              (C64, C64, C64, C32)]
    for at, xt, yt, compute in combos:
        t = f"A {at} x {xt} y {yt} compute {compute}"
        for opname, opA in OPS.items():
            for aname, alg in ALGS.items():
                kw = dict(type=t, opA=opname, alg=aname)
                kw.update(one(at, xt, yt, compute, opA, alg))
                out.append(kw)
                print(json.dumps(kw), flush=True)
    api.cusparseDestroy(h)
    return out


def quick_rehearsal():
    """the host logic at a tiny size on the CPU: byte model, error measure, the NATIVE predicate; timing needs a GPU"""
    assert bytes_moved(3, 4, 5, NT) == 16 + 100 + 64 + 48
    assert bytes_moved(3, 4, 5, TR, True) == 16 + 100 + 48 + 128
    y = torch.tensor([1 + 1j, 2j], dtype=torch.complex128)
    assert rel_err(y, y, torch.ones(2, dtype=torch.float64)) == 0.0
    assert eval(NATIVE)(NT, 1 << 20, 1 << 20, 16 << 20) in (True, False)
    print("# quick: host logic OK", flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--quick", action="store_true", help="CPU rehearsal of the host logic, then R-MAT 1M only")
    ap.add_argument("--status", action="store_true", help="also print the closed library's status grid")
    ap.add_argument("--only-status", action="store_true")
    ap.add_argument("--matrices", default=",".join(MATRICES))
    ap.add_argument("--ops", default="N,T,C")
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
        rows, cols, off, col, vals = matrix(mname)
        for opname in args.ops.split(","):
            for beta in (0j, BETA):
                rows_out.append(run_case(mname, rows, cols, off, col, vals, OPS[opname], beta, variants=variants))
                print(json.dumps(rows_out[-1]), flush=True)
        del off, col, vals
        torch.cuda.empty_cache()
    print(f"# {len(rows_out)} cases in {time.time() - t0:.0f} s on {name}", flush=True)
    if args.json:
        with open(args.json, "w") as f:
            json.dump(dict(card=name, rows=rows_out, status=status), f, indent=1)


if __name__ == "__main__":
    main()
