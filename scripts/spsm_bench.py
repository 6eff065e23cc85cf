"""Times the CSR triangular solve with many right-hand sides -- b200spsm_csr_solve (this build's level-ordered kernel, called
through its native entry point) against the closed cusparseSpSM_solve on the same buffers -- on one GPU and prints one JSON line.

Cases: spsv_bench.py's (the 5-point pattern of cuSPARSE/cg at 700^2, L and L^T, and at 4096^2, L; a bidiagonal chain of 2^16 rows;
a diagonal-only matrix of 2^24 rows) and the lower triangle of R-MAT 1M (16 per row, libb200gen.so) with its diagonal; all
NON_UNIT, diagonally dominant.  nrhs 1, 8, 32 and 128; B and C both column-major or both row-major; fp64 and fp32; host alpha.
Each solve is timed with CUDA events over back-to-back calls after warm-up (about --phase-ms per phase); each analysis once with a
host clock around it and a device synchronise.  Ours and the closed library's C are compared on every case.  At nrhs = 1, fp64,
column-major, our SpSV (libb200spsv.so) is timed too.  The card name and power limit are read in the same run.

    python scripts/spsm_bench.py [--phase-ms 300] [--cases stencil5_700,...]
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

from cudalibrarysamples_b200 import cusparse_api as cs  # noqa: E402
from cudalibrarysamples_b200 import lib as _lib  # noqa: E402
from cudalibrarysamples_b200 import workloads as W  # noqa: E402
from oracle import spsv_ref as R  # noqa: E402

NRHS = (1, 8, 32, 128)
ROW, COL = cs.CUSPARSE_ORDER_ROW, cs.CUSPARSE_ORDER_COL


def card():
    name = torch.cuda.get_device_name(0)
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                            capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:
        pl = ""
    return name, pl


def dominant(off, col, seed):
    rows = off.size - 1
    v = np.random.default_rng(seed).uniform(0.1, 1.0, int(off[-1]))
    r = np.repeat(np.arange(rows), np.diff(off))
    d = col == r
    v[d] = 0
    v[d] = (1.0 + np.bincount(r, weights=np.abs(v), minlength=rows))[r[d]]
    return v


def rmat_lower(rows):
    off, col, _ = W.rmat_csr(rows, avg_nnz=16, seed=42, val_seed=43)
    off, col = off.cpu().numpy().astype(np.int64), col.cpu().numpy().astype(np.int64)
    r = np.repeat(np.arange(rows), np.diff(off))
    keep = col < r
    return R.coo_to_csr(rows, np.concatenate([r[keep], np.arange(rows)]), np.concatenate([col[keep], np.arange(rows)]))


def cases(names):
    out = []
    for label, fn, ops in (("stencil5_700", lambda: R.stencil5_pattern(700), ("L", "Lt")),
                           ("stencil5_4096", lambda: R.stencil5_pattern(4096), ("L",)),
                           ("chain_64K", lambda: R.chain_pattern(1 << 16), ("L",)),
                           ("diagonal_16M", lambda: R.diagonal_pattern(1 << 24), ("L",)),
                           ("rmat_1M_lower", lambda: rmat_lower(1 << 20), ("L",))):
        if names and label not in names:
            continue
        out.append((label, fn, ops))
    return out


def time_calls(fn, phase_ms):
    """Mean ms per call of fn, after warm-up, over about phase_ms of back-to-back calls (CUDA events)."""
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    fn()
    b.record()
    torch.cuda.synchronize()
    one = max(a.elapsed_time(b), 1e-3)
    n = max(1, min(200, int(phase_ms / one)))
    for _ in range(min(n, 5)):
        fn()
    torch.cuda.synchronize()
    a.record()
    for _ in range(n):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / n, n


def run_case(L, rows, arr, nnz, op, nrhs, order, dtype, phase_ms, levels_out):
    tdt = torch.float64 if dtype == np.float64 else torch.float32
    code = 1 if dtype == np.float64 else 0
    tr = int(op == cs.CUSPARSE_OPERATION_TRANSPOSE)
    ld = rows if order == COL else nrhs
    B = torch.rand(rows * nrhs, dtype=tdt, device="cuda")
    Cours = torch.zeros_like(B)
    Cref = torch.zeros_like(B)
    sci, scj = (1, ld) if order == COL else (ld, 1)
    val = arr["val"] if arr["val"].dtype == tdt else arr["val"].to(tdt)
    # ours: the native entry points
    ws = torch.empty(L.b200spsm_csr_workspace_bytes(rows, nnz, tr), dtype=torch.uint8, device="cuda")
    lev = C.c_int64(0)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    assert L.b200spsm_csr_analysis(torch.cuda.current_stream().cuda_stream, rows, nnz, arr["off"].data_ptr(), arr["col"].data_ptr(), 0, 1, 0,
                                   tr, ws.data_ptr(), None, C.addressof(lev)) == 0
    an_ours = (time.perf_counter() - t0) * 1e3
    levels_out.append(lev.value)
    alpha = (C.c_double if code else C.c_float)(1.0)
    st = torch.cuda.current_stream().cuda_stream

    def ours():
        L.b200spsm_csr_solve(st, code, rows, nnz, 0, val.data_ptr(), None, C.addressof(alpha), 0, nrhs, B.data_ptr(), sci, scj,
                             Cours.data_ptr(), sci, scj, ws.data_ptr())
    ms_ours, n_ours = time_calls(ours, phase_ms)
    err_word = int(ws[8:12].view(torch.int32).item())
    # closed: the same B, its own C buffer, through the real library's SpSM
    api = cs.Api("cusparse")
    carr = dict(off=arr["off"], col=arr["col"], val=val)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    s = cs.SpSMSolver(api, rows, carr, B, Cref, nrhs, op_a=op, order_b=order, order_c=order)
    torch.cuda.synchronize()
    an_ref = (time.perf_counter() - t0) * 1e3          # descriptors + bufferSize + allocation + analysis
    fn = api.real.cusparseSpSM_solve
    argv = (s.handle, C.c_int(op), C.c_int(0), C.cast(C.pointer(alpha), C.c_void_p), s.mat, s.matB, s.matC, C.c_int(code), C.c_int(0),
            s.descr)

    def ref():
        fn(*argv)
    ms_ref, n_ref = time_calls(ref, phase_ms)
    s.close()
    a, b = Cours.double(), Cref.double()
    err = float(torch.linalg.norm(a - b) / max(float(torch.linalg.norm(b)), 1e-300))
    return dict(us_b200=round(ms_ours * 1e3, 2), us_cusparse=round(ms_ref * 1e3, 2), speedup=round(ms_ref / ms_ours, 3),
                analysis_ms_b200=round(an_ours, 2), analysis_ms_cusparse=round(an_ref, 2), rel_err=err, error_word=err_word,
                reps_b200=n_ours, reps_cusparse=n_ref)


def spsv_time(rows, arr, op, phase_ms):
    api = cs.Api("b200")
    s = cs.SpSVSolver(api, rows, arr, op=op)
    x = torch.rand(rows, dtype=torch.float64, device="cuda")
    y = torch.empty_like(x)
    s.api.cusparseDnVecSetValues(s.vecX, x)
    s.api.cusparseDnVecSetValues(s.vecY, y)
    one = C.c_double(1.0)
    fn = _lib.spsv().cusparseSpSV_solve
    argv = (s.handle, C.c_int(op), C.cast(C.pointer(one), C.c_void_p), s.mat, s.vecX, s.vecY, C.c_int(cs.CUDA_R_64F), C.c_int(0), s.descr)
    ms, n = time_calls(lambda: fn(*argv), phase_ms)
    s.close()
    return round(ms * 1e3, 2)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--phase-ms", type=float, default=300.0)
    ap.add_argument("--cases", default="")
    args = ap.parse_args()
    name, pl = card()
    L = _lib.shim()
    out = []
    tol = {np.float64: 1e-9, np.float32: 1e-3}
    for label, fn, ops in cases(set(filter(None, args.cases.split(",")))):
        off, col = fn()
        rows, nnz = off.size - 1, int(off[-1])
        arr = dict(off=torch.tensor(off, device="cuda"), col=torch.tensor(col, device="cuda"),
                   val=torch.tensor(dominant(off, col, 1), device="cuda"))
        for opname in ops:
            op = cs.CUSPARSE_OPERATION_TRANSPOSE if opname == "Lt" else cs.CUSPARSE_OPERATION_NON_TRANSPOSE
            spsv_us = None
            for dtype in (np.float64, np.float32):
                for order in (COL, ROW):
                    for nrhs in NRHS:
                        lv = []
                        rec = dict(case=f"{label}_{opname}", rows=rows, nnz=nnz, dtype="fp64" if dtype == np.float64 else "fp32",
                                   layout="row" if order == ROW else "col", nrhs=nrhs)
                        try:
                            rec.update(run_case(L, rows, arr, nnz, op, nrhs, order, dtype, args.phase_ms, lv))
                            rec["levels"] = lv[0]
                            rec["ok"] = rec["rel_err"] < tol[dtype] and rec["error_word"] == 0
                        except Exception as e:            # out of memory at the largest shapes: recorded, not hidden
                            rec["skipped"] = f"{type(e).__name__}: {str(e)[:120]}"
                            torch.cuda.empty_cache()
                        if nrhs == 1 and dtype == np.float64 and order == COL and "skipped" not in rec:
                            spsv_us = spsv_time(rows, arr, op, args.phase_ms)
                            rec["us_spsv_b200"] = spsv_us
                        out.append(rec)
                        print(json.dumps(rec), file=sys.stderr, flush=True)
        del arr
        torch.cuda.empty_cache()
    print(json.dumps(dict(bench="spsm_csr", gpu=name, power_limit_w=pl, phase_ms=args.phase_ms, cases=out)))


if __name__ == "__main__":
    main()
