#!/usr/bin/env python
"""Incomplete LU / Cholesky factorizations, ours (ilu0_csr.cu through the shim, B200SPMV_ILU0=on) against the closed library on the
same buffers, in one process (DESIGN.md 3.26).

Cases: cg's 5-point 700^2 (IC), bicgstab's 700^2 (ILU), a 5-point 4096^2, a diagonally dominant R-MAT 1M, the lower bidiagonal chain
of 2^16 rows and the diagonal of 2^24 rows (both kinds), each in fp32 and fp64.  The chain and the diagonal bound the cost of one
level barrier and of a row without dependencies.

Each side creates its own info and buffer (bufferSize, then analysis), and the same values are restored before every factorization,
outside the timed window.  Analysis and factorization are timed separately with CUDA events after a warm-up, median of --iters calls,
--repeat times per side alternating.  Reported: both medians, the speed-ups (ours / closed, per repeat), the levels, the largest
relative difference of the two factors, and b200ilu0_route's verdict.  The card's name and power limit are read in the same run.
usage: python scripts/ilu0_bench.py [--quick] [--iters N] [--warm N] [--repeat N] [--cases 700,chain,...] [--json out.json]"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from cudalibrarysamples_b200 import cusparse_api as cs  # noqa: E402
from oracle import ilu0_ref as R  # noqa: E402
from oracle import oracle as O  # noqa: E402


def native(kind, vtype, rows, nnz, levels):
    """The classes measured at least at parity in both repeats (DESIGN.md 3.26): the same predicate as ilu0_measured_native in
    csrc/cusparse_shim.cpp.  kind 0 = LU, 1 = IC; vtype 0 = fp32, 1 = fp64."""
    return False


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def cases(quick):
    g = 300 if quick else 4096
    out = [("cg 5-pt 700^2", ["ic"], lambda: O.gen_stencil5(700)),
           ("bicgstab 700^2", ["lu"], lambda: O.gen_stencil5(700, mass=0.3, ux=0.3, uy=0.2)),
           (f"5-pt {g}^2", ["ic", "lu"], lambda: O.gen_stencil5(g))]

    def rmat():
        n = 1 << (16 if quick else 20)
        off, col, _ = O.rmat_csr(n, avg_nnz=8, seed=21, val_seed=22)
        off, col = R.with_diagonal(off, col, n)
        return off, col, R.dominant(off, col, np.float64, 23)

    def chain():
        off, col = R.chain(1 << 16)
        return off, col, R.dominant(off, col, np.float64, 24)

    def diagonal():
        off, col = R.diagonal(1 << (20 if quick else 24))
        return off, col, np.linspace(0.5, 4.0, off.size - 1)
    out += [("R-MAT %s dominant" % ("64K" if quick else "1M"), ["ic", "lu"], rmat), ("chain 2^16", ["ic", "lu"], chain),
            ("diagonal 2^%d" % (20 if quick else 24), ["ic", "lu"], diagonal)]
    return out


class Side:
    """One implementation's handle, descriptor, info and buffer for one matrix: analysis and factorization timed separately."""

    def __init__(self, api, kind, dtype, m, offd, cold, v0):
        self.api, self.kind, self.m, self.offd, self.cold, self.v0 = api, kind, m, offd, cold, v0
        self.t = "S" if dtype == torch.float32 else "D"
        self.name = "csric02" if kind == "ic" else "csrilu02"
        self.v = v0.clone()
        self.h = api.cusparseCreate()
        self.descr, self.info = C.c_void_p(), C.c_void_p()
        api._call(api.real, "cusparseCreateMatDescr", C.byref(self.descr))
        api._call(api.lib, "cusparseCreate%sInfo" % ("Csric02" if kind == "ic" else "Csrilu02"), C.byref(self.info))
        size = C.c_int()
        api._call(api.lib, f"cusparse{self.t}{self.name}_bufferSize", *self.args(), C.byref(size))
        self.buf = torch.empty(max(size.value, 16), dtype=torch.uint8, device="cuda")

    def args(self):
        return (self.h, C.c_int(self.m), C.c_int(self.cold.numel()), self.descr, cs._ptr(self.v), cs._ptr(self.offd), cs._ptr(self.cold),
                self.info)

    def analysis(self):
        self.api._call(self.api.lib, f"cusparse{self.t}{self.name}_analysis", *self.args(), C.c_int(1), cs._ptr(self.buf))

    def factor(self):
        self.api._call(self.api.lib, f"cusparse{self.t}{self.name}", *self.args(), C.c_int(1), cs._ptr(self.buf))

    def time(self, what, iters, warm=2):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        ts = []
        for it in range(warm + iters):
            if what == "factor":
                self.v.copy_(self.v0)
                torch.cuda.synchronize()
            e0.record()
            self.analysis() if what == "analysis" else self.factor()
            e1.record()
            torch.cuda.synchronize()
            if it >= warm:
                ts.append(e0.elapsed_time(e1) * 1e3)
        return float(np.median(ts))

    def close(self):
        api = self.api
        api._call(api.lib, "cusparseDestroy%sInfo" % ("Csric02" if self.kind == "ic" else "Csrilu02"), self.info)
        api._call(api.real, "cusparseDestroyMatDescr", self.descr)
        api.cusparseDestroy(self.h)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--quick", action="store_true")
    ap.add_argument("--iters", type=int, default=7)
    ap.add_argument("--repeat", type=int, default=2)
    ap.add_argument("--cases", default="", help="comma-separated substrings of the case labels to run (default: all)")
    ap.add_argument("--warm", type=int, default=2, help="untimed calls before each timed window")
    ap.add_argument("--json", default="")
    a = ap.parse_args()
    gpu = card()
    print(f"# {gpu}")
    ours, closed = cs.Api("b200"), cs.Api("cusparse")
    rows_out = []
    for label, kinds, make in cases(a.quick):
        if a.cases and not any(c in label for c in a.cases.split(",")):
            continue
        off, col, val = make()
        off, col = np.asarray(off, np.int32), np.asarray(col, np.int32)
        m, nnz = off.size - 1, col.size
        offd, cold = torch.tensor(off, device="cuda"), torch.tensor(col, device="cuda")
        for dtype in (torch.float32, torch.float64):
            v0 = torch.tensor(np.asarray(val), dtype=dtype, device="cuda")
            for kind in kinds:
                ours.set_option("B200SPMV_ILU0", "on")
                sides = {"ours": Side(ours, kind, dtype, m, offd, cold, v0), "closed": Side(closed, kind, dtype, m, offd, cold, v0)}
                ta = {k: [] for k in sides}
                tf = {k: [] for k in sides}
                for _ in range(a.repeat):
                    for k, s in sides.items():
                        ta[k].append(s.time("analysis", a.iters, a.warm))
                        tf[k].append(s.time("factor", a.iters, a.warm))
                lev = C.c_int64(-1)
                ws = sides["ours"].buf
                ours.lib.b200ilu0_analysis(torch.cuda.current_stream().cuda_stream, m, nnz, offd.data_ptr(), cold.data_ptr(), 0,
                                           ws.data_ptr(), None, C.byref(lev))
                torch.cuda.synchronize()
                for s in sides.values():                      # one more factorization from the same values, then compare
                    s.v.copy_(v0)
                    s.analysis()
                    s.factor()
                torch.cuda.synchronize()
                x, y = sides["ours"].v.double(), sides["closed"].v.double()
                diff = float((x - y).abs().max() / y.abs().max())
                for s in sides.values():
                    s.close()
                ours.set_option("B200SPMV_ILU0", "auto")
                route = ours.lib.b200ilu0_route(1 if kind == "ic" else 0, 0 if dtype == torch.float32 else 1, m, nnz, lev.value)
                sa = [c / o for o, c in zip(ta["ours"], ta["closed"])]
                sf = [c / o for o, c in zip(tf["ours"], tf["closed"])]
                row = dict(case=label, kind=kind, dtype=str(dtype).split(".")[-1], rows=m, nnz=nnz, levels=lev.value,
                           analysis_us=dict(ours=ta["ours"], closed=ta["closed"]), factor_us=dict(ours=tf["ours"], closed=tf["closed"]),
                           speedup_analysis=sa, speedup_factor=sf, max_rel_diff=diff, route=route)
                rows_out.append(row)
                print(f"{label:22s} {kind} {row['dtype']:8s} levels {lev.value:8d} | analysis ours "
                      f"{'/'.join('%.0f' % t for t in ta['ours'])} closed {'/'.join('%.0f' % t for t in ta['closed'])} us "
                      f"x{'/'.join('%.2f' % s for s in sa)} | factor ours {'/'.join('%.0f' % t for t in tf['ours'])} closed "
                      f"{'/'.join('%.0f' % t for t in tf['closed'])} us x{'/'.join('%.2f' % s for s in sf)} | diff {diff:.1e} route {route}",
                      flush=True)
    if a.json:
        with open(a.json, "w") as f:
            json.dump(dict(card=gpu, rows=rows_out), f, indent=1)


if __name__ == "__main__":
    main()
