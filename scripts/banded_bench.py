#!/usr/bin/env python
"""Batched banded solves, ours (batched_banded.cu) against the closed library on the same buffers, in one process (DESIGN.md 3.25).

Shapes: m in {16, 64, 256, 1024, 4096} x batch in {1K, 16K, 256K} x fp32 / fp64 / complex64 / complex128 x {gpsv, gtsv algo 0, 1,
2}, skipping the shapes whose arrays (ours and the closed library's workspace) would pass --max-gb.  Diagonally dominant systems,
interleaved; the same diagonals and right-hand sides go to both sides, and the two solutions are compared once.  The closed library's
solves write some coefficient arrays, so each side solves on its own copy of them.  Every timed call of either side first restores x
and both copies, so the two totals carry the same copies; the speed-up is the ratio of the totals, with nothing subtracted (it lies
between 1 and the ratio of the solves alone).  The times and GB/s take the separately timed restore off.

Each call is timed with CUDA events after a warm-up, median of three windows, --repeat times per side alternating.  Reported per row: both times, the speed-up (median, and the range over the repeats), GB/s on
the compulsory bytes (the diagonals and the right-hand side read once, x written once) and on the bytes including our scratch
traffic (the factor written and read back, x written twice and read twice; an upper bound on the HBM traffic, since part of it
is served from L2), each also as a share of 3.35 TB/s, the largest relative
difference of the two solutions, and b200banded_route's verdict.  The card's name, power limit and SM clock are read in the same run.
usage: python scripts/banded_bench.py [--quick] [--ms M,..] [--batches B,..] [--repeat N] [--max-gb G] [--json out.json]"""
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
from cudalibrarysamples_b200 import lib as _lib  # noqa: E402

DEV = torch.device("cuda:0")
PEAK = 3.35e12
DTYPES = (torch.float32, torch.float64, torch.complex64, torch.complex128)
VT = {torch.float32: 0, torch.float64: 1, torch.complex64: 4, torch.complex128: 5}
T = {torch.float32: "S", torch.float64: "D", torch.complex64: "C", torch.complex128: "Z"}
# (name, op for b200banded_route, algo, sub-diagonals P, our factor entries per row W)
METHODS = (("gpsv", 0, 0, 2, 4), ("gtsv0", 1, 0, 1, 1), ("gtsv1", 1, 1, 1, 2), ("gtsv2", 1, 2, 1, 2))

# The classes b200banded_route runs natively (DESIGN.md 3.25; BANDED_PARITY in cusparse_shim.cpp holds the same bits): on the grid
# m in NATIVE_M x batch in NATIVE_BATCH, bit (ib * 4 + im) of NATIVE_GRID[method][type] is set where that point ran at least at
# parity with the closed library in both repeats (method: gpsv, gtsv algo 0, 1, 2; type: fp32, fp64, complex64, complex128).  Between
# grid points a call is native when every corner of its cell is; everything off the grid is forwarded.
NATIVE_M = (64, 256, 1024, 4096)
NATIVE_BATCH = (16384, 65536, 262144, 1048576)
NATIVE_GRID = [[14208, 4960, 4608, 4976], [14335, 14335, 2047, 4464], [14080, 4976, 4928, 4976], [14080, 4976, 4960, 4976]]
_TYPE = {0: 0, 1: 1, 4: 2, 5: 3}


def _bracket(grid, v):
    if v < grid[0] or v > grid[-1]:
        return None
    i = max(k for k, g in enumerate(grid) if g <= v)
    return (i, i) if grid[i] == v else (i, i + 1)


def native(op, vtype, algo, m, batch):
    """b200banded_route's measured classes for an admitted call (op 0 gpsv / 1 gtsv, vtype a cudaDataType)"""
    bm, bb = _bracket(NATIVE_M, m), _bracket(NATIVE_BATCH, batch)
    if bm is None or bb is None or vtype not in _TYPE:
        return False
    bits = NATIVE_GRID[0 if op == 0 else 1 + algo][_TYPE[vtype]]
    return all(bits >> (ib * 4 + im) & 1 for ib in bb for im in bm)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name(0)


def timeit(fn, budget=0.03):
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


def operands(m, batch, P, dt, seed):
    """diagonally dominant diagonals (sub-diagonals first) and right-hand sides, (m, batch), on the device"""
    g = torch.Generator(device=DEV).manual_seed(seed)
    rdt = torch.float32 if dt in (torch.float32, torch.complex64) else torch.float64

    def draw():
        v = torch.rand(m, batch, device=DEV, generator=g, dtype=rdt) * 2 - 1
        if dt.is_complex:
            v = torch.complex(v, torch.rand(m, batch, device=DEV, generator=g, dtype=rdt) * 2 - 1)
        return v.to(dt)

    diags = [draw() for _ in range(2 * P + 1)]
    diags[P] = diags[P] + (2 * P + 1.5)
    return diags, draw()


def closed_solve(R, h, name, dt, algo, m, batch, diags, x, buf):
    fn = getattr(R, f"cusparse{T[dt]}{name}")
    st = fn(h, C.c_int(algo), C.c_int(m), *[C.c_void_p(d.data_ptr()) for d in diags], C.c_void_p(x.data_ptr()), C.c_int(batch),
            C.c_void_p(buf.data_ptr()))
    if st != 0:
        raise RuntimeError(f"cusparse{T[dt]}{name} -> {st}")


def closed_buffer(R, h, name, dt, algo, m, batch, diags, x):
    size = C.c_size_t()
    st = getattr(R, f"cusparse{T[dt]}{name}_bufferSizeExt")(h, C.c_int(algo), C.c_int(m), *[C.c_void_p(d.data_ptr()) for d in diags],
                                                           C.c_void_p(x.data_ptr()), C.c_int(batch), C.byref(size))
    if st != 0:
        raise RuntimeError(f"bufferSizeExt -> {st}")
    return size.value


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--quick", action="store_true", help="m 64 / 1024, batch 16K only")
    ap.add_argument("--max-gb", type=float, default=30.0)
    ap.add_argument("--json", default="")
    ap.add_argument("--ms", default="", help="comma-separated m values instead of the default grid")
    ap.add_argument("--batches", default="", help="comma-separated batch counts instead of the default grid")
    ap.add_argument("--repeat", type=int, default=2, help="timings per side and shape, alternating; the median is reported")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("banded_bench.py measures on the GPU; there is none here")
    L = _lib.shim()
    api = cs.Api("cusparse")
    R = api.real
    h = api.cusparseCreate()
    stream = torch.cuda.current_stream().cuda_stream
    api.cusparseSetStream(h, stream)
    ms = (64, 1024) if a.quick else (16, 64, 256, 1024, 4096)
    batches = (16384,) if a.quick else (1024, 16384, 262144)
    if a.ms:
        ms = tuple(int(v) for v in a.ms.split(","))
    if a.batches:
        batches = tuple(int(v) for v in a.batches.split(","))
    gpu = card()
    print(f"# {gpu}", flush=True)
    rows = []
    for name, op, algo, P, W in METHODS:
        cname = "gpsvInterleavedBatch" if op == 0 else "gtsvInterleavedBatch"
        for dt in DTYPES:
            w = torch.empty(0, dtype=dt).element_size()
            for m in ms:
                for batch in batches:
                    n = m * batch
                    ours_ws = (L.b200gpsv_interleaved_workspace_bytes(VT[dt], m, batch) if op == 0 else
                               L.b200gtsv_interleaved_workspace_bytes(VT[dt], algo, m, batch))
                    # diagonals + both sides' copies, x + b, our workspace, the closed one (~ ours)
                    est = (3 * (2 * P + 1) + 2) * n * w + 2 * ours_ws
                    if est > a.max_gb * 1e9:
                        continue
                    diags, b = operands(m, batch, P, dt, seed=m + batch)
                    cdiags = [d.clone() for d in diags]
                    x = b.clone()
                    cbuf = torch.empty(max(closed_buffer(R, h, cname, dt, algo, m, batch, cdiags, x), 16), dtype=torch.uint8, device=DEV)
                    obuf = torch.empty(max(ours_ws, 16), dtype=torch.uint8, device=DEV)

                    odiags = [d.clone() for d in diags]

                    def restore():
                        x.copy_(b)
                        for o, c, d in zip(odiags, cdiags, diags):
                            o.copy_(d)
                            c.copy_(d)

                    def ours():
                        restore()
                        rc = (L.b200gpsv_interleaved(stream, VT[dt], m, *[d.data_ptr() for d in odiags], x.data_ptr(), batch, obuf.data_ptr())
                              if op == 0 else
                              L.b200gtsv_interleaved(stream, VT[dt], algo, m, *[d.data_ptr() for d in odiags], x.data_ptr(), batch,
                                                     obuf.data_ptr()))
                        assert rc == 0, rc

                    def closed():
                        restore()
                        closed_solve(R, h, cname, dt, algo, m, batch, cdiags, x, cbuf)

                    ours(); torch.cuda.synchronize()
                    xo = x.clone()
                    closed(); torch.cuda.synchronize()
                    xc = x.clone()
                    diff = float(((xo - xc).abs().max() / xc.abs().max().clamp_min(1e-30)).item())
                    del xo, xc
                    # Both timed calls first restore the same inputs (x and both sides' coefficient copies), so each solve starts from
                    # the same values and both totals carry the same copies.  The speed-up is the ratio of the totals, nothing
                    # subtracted: it lies between 1 and the solves' own ratio.  Only the GB/s take the separately timed copies off.
                    ts_o, ts_c, ts_r = [], [], []
                    for _ in range(a.repeat):
                        ts_o.append(timeit(ours))
                        ts_c.append(timeit(closed))
                        ts_r.append(timeit(restore))
                    T_o, T_c, t_r = float(np.median(ts_o)), float(np.median(ts_c)), float(np.median(ts_r))
                    speedups = [c / o for o, c in zip(ts_o, ts_c)]
                    t_o, t_c = max(T_o - t_r, 1e-9), max(T_c - t_r, 1e-9)
                    compulsory = (2 * P + 3) * n * w
                    scratch = (2 * P + 2 * W + 5) * n * w
                    r = dict(method=name, dtype=str(dt).replace("torch.", ""), m=m, batch=batch, ours_us=t_o * 1e6, closed_us=t_c * 1e6,
                             speedup=T_c / T_o, speedup_min=min(speedups), speedup_max=max(speedups), ours_gbs=compulsory / t_o / 1e9, ours_gbs_scratch=scratch / t_o / 1e9,
                             closed_gbs=compulsory / t_c / 1e9, ours_peak=compulsory / t_o / PEAK,
                             ours_peak_scratch=scratch / t_o / PEAK, rel_diff=diff, workspace_ours=ours_ws, workspace_closed=cbuf.numel(),
                             routed=bool(native(op, VT[dt], algo, m, batch)))
                    rows.append(r)
                    print(f"{name:6s} {r['dtype']:10s} m={m:5d} batch={batch:7d}  ours {r['ours_us']:10.1f} us  closed {r['closed_us']:10.1f} us"
                          f"  x{r['speedup']:5.2f} ({r['speedup_min']:4.2f}-{r['speedup_max']:4.2f})  {r['ours_gbs']:7.1f} GB/s ({100 * r['ours_peak']:4.1f} %)  incl. scratch"
                          f" {r['ours_gbs_scratch']:7.1f} GB/s ({100 * r['ours_peak_scratch']:4.1f} %)  closed {r['closed_gbs']:7.1f} GB/s"
                          f"  diff {diff:.1e}  ws {ours_ws >> 10} / {cbuf.numel() >> 10} KiB  {'native' if r['routed'] else 'forwarded'}",
                          flush=True)
                    del diags, cdiags, b, x, cbuf, obuf
                    torch.cuda.empty_cache()
    api.cusparseDestroy(h)
    if a.json:
        with open(a.json, "w") as f:
            json.dump(dict(card=gpu, rows=rows), f, indent=1)


if __name__ == "__main__":
    main()
