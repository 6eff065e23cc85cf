"""Times the CSR triangular solve (cusparseSpSV_solve) of libb200spsv.so against the closed libcusparse on one GPU and
prints one JSON line.

Cases: the lower-triangle solve L and the transposed solve L^T on the 5-point pattern of cuSPARSE/cg (both triangles
stored, as cg's matL) at 700^2 (1399 dependency levels) and at 4096^2, a bidiagonal chain of 2^16 rows (every row depends
on the one before), and a diagonal-only matrix of 2^24 rows (no dependencies).  fp64, host alpha.  Each solve is timed with CUDA events over
--reps back-to-back calls after --warmup calls (both fewer when one call is slow: about 2 s per phase); the card name and power limit are queried in the same run.

    python scripts/spsv_bench.py [--reps 50] [--warmup 10]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

from cudalibrarysamples_b200 import cusparse_api as cs  # noqa: E402
from oracle import oracle as O  # noqa: E402
from oracle import spsv_ref as R  # noqa: E402


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
    v = O.uniform(seed, int(off[-1]), np.float64)
    r = np.repeat(np.arange(rows), np.diff(off))
    d = col == r
    v[d] = 0
    v[d] = (1.0 + np.bincount(r, weights=np.abs(v), minlength=rows))[r[d]]
    return v


def time_solve(impl, rows, arr, op, reps, warmup):
    api = cs.Api(impl)
    s = cs.SpSVSolver(api, rows, arr, fill=cs.CUSPARSE_FILL_MODE_LOWER, diag=cs.CUSPARSE_DIAG_TYPE_NON_UNIT, op=op)
    x = torch.ones(rows, dtype=torch.float64, device="cuda")
    y = torch.empty_like(x)
    s.api.cusparseDnVecSetValues(s.vecX, x)
    s.api.cusparseDnVecSetValues(s.vecY, y)
    import ctypes as C
    one = C.c_double(1.0)
    fn = s.api.sv.cusparseSpSV_solve
    argv = (s.handle, C.c_int(op), C.cast(C.pointer(one), C.c_void_p), s.mat, s.vecX, s.vecY, C.c_int(cs.CUDA_R_64F),
            C.c_int(cs.CUSPARSE_SPSV_ALG_DEFAULT), s.descr)
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    assert fn(*argv) == 0                                                       # first warm-up call, timed to pace the rest
    b.record()
    torch.cuda.synchronize()
    budget = max(1, int(2000.0 / max(a.elapsed_time(b), 1e-3)))                # about 2 s per phase when one call is slow
    for _ in range(min(warmup, budget) - 1):
        assert fn(*argv) == 0
    torch.cuda.synchronize()
    reps = min(reps, budget)
    a.record()
    for _ in range(reps):
        fn(*argv)
    b.record()
    torch.cuda.synchronize()
    out = y.cpu().numpy()
    s.close()
    return a.elapsed_time(b) / reps * 1e3, out, reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    args = ap.parse_args()
    name, pl = card()
    cases = []
    for label, (off, col) in (("stencil5_700", R.stencil5_pattern(700)), ("stencil5_4096", R.stencil5_pattern(4096)),
                              ("chain_64K", R.chain_pattern(1 << 16)), ("diagonal_16M", R.diagonal_pattern(1 << 24))):
        rows = off.size - 1
        arr = dict(off=torch.tensor(off, device="cuda"), col=torch.tensor(col, device="cuda"),
                   val=torch.tensor(dominant(off, col, 1), device="cuda"))
        for opname, op in (("L", cs.CUSPARSE_OPERATION_NON_TRANSPOSE), ("Lt", cs.CUSPARSE_OPERATION_TRANSPOSE)):
            if label.startswith("diagonal") and op == cs.CUSPARSE_OPERATION_TRANSPOSE:
                continue
            us_ours, y_ours, n_ours = time_solve("b200", rows, arr, op, args.reps, args.warmup)
            us_ref, y_ref, n_ref = time_solve("cusparse", rows, arr, op, args.reps, args.warmup)
            err = float(np.linalg.norm(y_ours - y_ref) / np.linalg.norm(y_ref))
            cases.append(dict(case=f"{label}_{opname}", rows=rows, nnz=int(off[-1]), us_b200=round(us_ours, 2),
                              us_cusparse=round(us_ref, 2), speedup=round(us_ref / us_ours, 3), rel_err=err, reps_b200=n_ours,
                              reps_cusparse=n_ref))
            print(f"{label:15s} {opname:2s}  ours {us_ours:10.1f} us   cusparse {us_ref:10.1f} us   x{us_ref / us_ours:6.2f}  "
                  f"rel err {err:.1e}", file=sys.stderr, flush=True)
    print(json.dumps(dict(bench="spsv_csr_fp64", gpu=name, power_limit_w=pl, reps=args.reps, warmup=args.warmup, cases=cases)))


if __name__ == "__main__":
    main()
