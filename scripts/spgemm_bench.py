#!/usr/bin/env python
"""cusparseSpGEMMreuse_compute: b200spgemm_compute (B200SPMV_SPGEMM=on) against the closed library on the same device arrays
(DESIGN.md 3.28).  Each side has its own SpGEMM descriptor and buffers.

Per workload: the hot path, reuse_compute (CUDA events around `calls` back-to-back calls after a warm-up, the two sides alternating
over `repeats` rounds, the median per call), and the one-time set-up of the sample's sequence (workEstimation, nnz, copy; ours also
builds the plan inside reuse_copy), host clock around a synchronised run.  The outputs must agree to 1e-5 (fp32) / 1e-12 (fp64)
relative error.  Bytes moved and products per second come from the shapes (oracle/spgemm_ref.py).  The card name and power limit
are read in the same run.  NATIVE is the predicate of the classes the shim routes natively by default.

usage: python scripts/spgemm_bench.py [--quick] [--repeats N] [--calls N] [--json out.json]"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import scipy.sparse as sp
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from cudalibrarysamples_b200 import cusparse_api as cs  # noqa: E402
from oracle import spgemm_ref as R  # noqa: E402


def NATIVE(workload, dtype):
    """The classes measured at least at parity with the closed reuse_compute: none so far (the shim's spgemm_measured_native)."""
    return False


def workloads(quick):
    s5, s7, u, rm, g = (256, 32, 1 << 16, 14, 256) if quick else (2048, 128, 1 << 20, 18, 2048)
    A5 = sp.csr_matrix(R.stencil5(s5)[::-1])
    A7 = sp.csr_matrix(R.stencil7(s7)[::-1])
    Au = sp.csr_matrix(R.uniform(u, 8, 1)[::-1], shape=(u, u))
    Ar = sp.csr_matrix(R.rmat(rm, 8, 2)[::-1], shape=(1 << rm, 1 << rm))
    Rg = sp.csr_matrix(R.restriction2(g)[::-1], shape=((g // 2) ** 2, g * g))
    Ag = A5 if g == s5 else sp.csr_matrix(R.stencil5(g)[::-1])
    return [(f"stencil5 {s5}^2 A.A", A5, A5, (torch.float32, torch.float64)),
            (f"stencil7 {s7}^3 A.A", A7, A7, (torch.float32, torch.float64)),
            (f"uniform {u} x 8 A.A", Au, Au, (torch.float64,)),
            (f"rmat 2^{rm} x 8 A.A", Ar, Ar, (torch.float64,)),
            (f"restriction 2:1 of {g}^2 R.A", Rg, Ag, (torch.float64,))]


def dev(M, dtype):
    d = torch.device("cuda")
    return dict(rows=M.shape[0], cols=M.shape[1], off=torch.tensor(M.indptr, dtype=torch.int32, device=d),
                col=torch.tensor(M.indices, dtype=torch.int32, device=d), val=torch.tensor(M.data, dtype=dtype, device=d))


def setup(api, A, B, dtype):
    torch.cuda.synchronize()
    t = time.perf_counter()
    r = cs.SpGEMMReuse(api, A, B)
    torch.cuda.synchronize()
    return r, time.perf_counter() - t


def time_calls(r, calls):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(calls):
        r.compute(1.0, 0.0)
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1) / calls * 1e-3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--quick", action="store_true", help="small sizes (a rehearsal, not a measurement)")
    ap.add_argument("--repeats", type=int, default=7)
    ap.add_argument("--calls", type=int, default=10)
    ap.add_argument("--json", default=None, help="also write the rows to this file")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("spgemm_bench.py measures on the GPU: no device found")
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip()
    ours_api, closed_api = cs.Api("b200"), cs.Api("cusparse")
    ours_api.set_option("B200SPMV_SPGEMM", "on")
    rows = []
    for name, MA, MB, dtypes in workloads(a.quick):
        for dtype in dtypes:
            A, B = dev(MA, dtype), dev(MB, dtype)
            theirs, t_setup_closed = setup(closed_api, A, B, dtype)
            ours, t_setup_ours = setup(ours_api, A, B, dtype)
            ours_api.reset_stats()
            x, y = ours.compute().double(), theirs.compute().double()
            err = (torch.linalg.norm(x - y) / torch.linalg.norm(y)).item()
            assert ours_api.stats()["native"] == 1, "the native path did not run"
            one = max(time_calls(r, 1) for r in (ours, theirs))           # warm-up, and the size of a timed window
            calls = max(1, min(a.calls, int(0.2 / one)))                    # about 0.2 s per side and round at most
            t_ours, t_closed = [], []
            for _ in range(a.repeats):
                t_ours.append(time_calls(ours, calls))
                t_closed.append(time_calls(theirs, calls))
            to, tc = statistics.median(t_ours), statistics.median(t_closed)
            vb = 4 if dtype == torch.float32 else 8
            prods = int(R.products_per_row(MA.indptr, MA.indices, MB.indptr).sum())
            byt = R.traffic_bytes(MA.shape[0], MA.nnz, MB.nnz, ours.nnz, prods, vb)
            row = dict(workload=name, dtype=str(dtype)[6:], rows=MA.shape[0], nnz_a=int(MA.nnz), nnz_b=int(MB.nnz), nnz_c=ours.nnz,
                       products=prods, calls=calls, ours_ms=to * 1e3, closed_ms=tc * 1e3, speedup=tc / to, ours_gbps=byt / to / 1e9,
                       ours_gprod_s=prods / to / 1e9, closed_gprod_s=prods / tc / 1e9, setup_ours_ms=t_setup_ours * 1e3,
                       setup_closed_ms=t_setup_closed * 1e3, rel_err=err, native_by_default=NATIVE(name, dtype), card=card)
            assert err < (1e-5 if dtype == torch.float32 else 1e-12), row
            rows.append(row)
            print(json.dumps(row), flush=True)
            ours.close(); theirs.close()
            del ours, theirs, A, B
            torch.cuda.empty_cache()
    if a.json:
        with open(a.json, "w") as f:
            json.dump(dict(card=card, quick=a.quick, rows=rows), f, indent=1)
    print(f"\n{card}")
    print("| workload | type | nnz(C) | products | ours ms | closed ms | closed / ours | ours GB/s | set-up ours / closed ms |")
    print("|---|---|---|---|---|---|---|---|---|")
    for r in rows:
        print(f"| {r['workload']} | {r['dtype']} | {r['nnz_c']} | {r['products']} | {r['ours_ms']:.3f} | {r['closed_ms']:.3f} | "
              f"{r['speedup']:.2f}x | {r['ours_gbps']:.0f} | {r['setup_ours_ms']:.1f} / {r['setup_closed_ms']:.1f} |")


if __name__ == "__main__":
    main()
