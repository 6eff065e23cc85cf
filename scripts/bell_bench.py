#!/usr/bin/env python
"""Blocked-ELL SpMM, ours (b200spmm_bell) against the closed library's cusparseSpMM on the same buffers (DESIGN.md 3.14).

M = K = 16384, random distinct block columns per block-row (seeded), alpha = 1, beta = 0.  Each side runs as a CUDA graph of
--calls products, timed with CUDA events after a warm-up, median of --reps replays.  Reported per case: us per product, TFLOP/s on
2 * (non-empty blocks) * bs^2 * N, effective GB/s on the compulsory bytes (ellColInd + ellValue + B once + C), which data-sheet bound
applies (989 TFLOP/s dense fp16 / bf16, 3.35 TB/s HBM3), and each side's largest error against an fp64 product.  The card's name and
power limit are read in the same run.
usage: python scripts/bell_bench.py [--quick | --small | --native-classes | --structures] [--json out.json]"""
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

PEAK_FLOPS = 989e12        # H100 SXM data sheet, dense fp16 / bf16 tensor
PEAK_BYTES = 3.35e12       # H100 SXM data sheet, HBM3
DEV = torch.device("cuda:0")
ROW, COL = cs.CUSPARSE_ORDER_ROW, cs.CUSPARSE_ORDER_COL
# (name, A / B type, C type, order of B and C)
KINDS = [("f16-col", torch.float16, torch.float16, COL), ("f16-row", torch.float16, torch.float16, ROW),
         ("bf16-f32-col", torch.bfloat16, torch.float32, COL)]
# with these two, every type combination and both orders the route can keep native (--native-classes)
MORE_KINDS = [("f16-f32-row", torch.float16, torch.float32, ROW), ("bf16-bf16-row", torch.bfloat16, torch.bfloat16, ROW)]


def structures(nb, eb, seed):
    """--structures: block-column layouts on which the closed library's result is compared with fp64 (every row stores eb blocks
    unless said otherwise; -1 = empty slot)"""
    rng = np.random.default_rng(seed)
    full = np.sort(np.array([rng.choice(nb, eb, replace=False) for _ in range(nb)]), axis=1)
    trailing, leading, empty_row = full.copy(), full.copy(), full.copy()
    trailing[:, -1] = -1                                   # -1 behind the stored blocks, ascending columns
    leading[:, 1:] = full[:, :-1]                          # -1 before the stored blocks, ascending columns
    leading[:, 0] = -1
    empty_row[::4] = -1                                    # every fourth block-row stores nothing, the others are full
    return {"full, ascending": full, "full, descending": full[:, ::-1].copy(), "-1 last, ascending": trailing,
            "-1 first, ascending": leading, "all-empty block-rows, others full": empty_row}


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name(0)


def make_case(m, k, bs, density, n, dt, ct, seed):
    nbr, nbc = m // bs, k // bs
    eb = max(1, int(round(density * nbc)))
    g = torch.Generator(device=DEV).manual_seed(seed)
    ci = torch.argsort(torch.rand(nbr, nbc, device=DEV, generator=g), dim=1)[:, :eb].sort(dim=1).values.to(torch.int32).contiguous()
    vals = (torch.rand(m, eb * bs, device=DEV, generator=g) * 2 - 1).to(dt)
    B = (torch.rand(k, n, device=DEV, generator=g) * 2 - 1).to(dt)
    return ci, vals, B, eb


def reference(ci, vals, B, bs, eb, m, n):
    """fp64 A @ B, one batched product per slot"""
    nbr = m // bs
    Bb = B.double().view(-1, bs, n)
    Av = vals.double().view(nbr, bs, eb, bs)
    out = torch.zeros(nbr, bs, n, dtype=torch.float64, device=DEV)
    for j in range(eb):
        live = (ci[:, j] >= 0).double().view(-1, 1, 1)
        out += torch.bmm(Av[:, :, j, :], Bb[ci[:, j].clamp(min=0).long()]) * live
    return out.view(m, n)


def graph_time(fn, calls, reps, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    try:
        return _graph_time(fn, calls, reps)
    except RuntimeError:                      # not capturable: the same loop, launched eagerly
        torch.cuda.synchronize()
        ts = []
        for _ in range(reps):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for _ in range(calls):
                fn()
            b.record()
            torch.cuda.synchronize()
            ts.append(a.elapsed_time(b) * 1e3 / calls)
        return float(np.median(ts))


def _graph_time(fn, calls, reps):
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    g = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s):
        with torch.cuda.graph(g, stream=s):
            for _ in range(calls):
                fn()
    torch.cuda.synchronize()
    g.replay()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        g.replay()
        b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b) * 1e3 / calls)
    return float(np.median(ts))


def run_case(m, k, bs, density, n, kind, calls, reps, warmup, seed=1, ci=None):
    name, dt, ct, order = kind
    if ci is None:
        ci, vals, B, eb = make_case(m, k, bs, density, n, dt, ct, seed)
    else:                                                  # a given structure (--structures)
        _, vals, B, eb = make_case(m, k, bs, ci.shape[1] / (k // bs), n, dt, ct, seed)
        ci = torch.tensor(ci, dtype=torch.int32, device=DEV)
    if order == ROW:
        Bs, ldb = B.contiguous().view(-1), n
    else:
        Bs, ldb = B.t().contiguous().view(-1), k
    ldc = n if order == ROW else m
    ref = reference(ci, vals, B, bs, eb, m, n)
    out = {}
    # ours: b200spmm_bell
    lib = _lib.shim()
    Co = torch.zeros(m * n, dtype=ct, device=DEV)
    al, be = C.c_float(1.0), C.c_float(0.0)
    tcode = {torch.float16: cs.CUDA_R_16F, torch.bfloat16: cs.CUDA_R_16BF, torch.float32: cs.CUDA_R_32F}

    def ours():
        rc = lib.b200spmm_bell(torch.cuda.current_stream().cuda_stream, tcode[dt], tcode[ct], m, k, n, bs, eb * bs, ci.data_ptr(),
                               vals.data_ptr(), 0, C.addressof(al), C.addressof(be), 0, Bs.data_ptr(), ldb, int(order == ROW),
                               Co.data_ptr(), ldc, int(order == ROW))
        assert rc == 0, rc
    out["ours_us"] = graph_time(ours, calls, reps, warmup)
    got = Co.view(m, n) if order == ROW else Co.view(n, m).t()
    out["ours_err"] = float((got.double() - ref).abs().max())
    # the closed library: cusparseSpMM on the same buffers
    api = cs.Api("cusparse")
    Cc = torch.zeros(m * n, dtype=ct, device=DEV)
    h = api.cusparseCreate()
    matA = api.cusparseCreateBlockedEll(m, k, bs, eb * bs, ci, vals)
    matB = api.cusparseCreateDnMat(k, n, ldb, Bs, order)
    matC = api.cusparseCreateDnMat(m, n, ldc, Cc, order)
    NT = cs.CUSPARSE_OPERATION_NON_TRANSPOSE
    try:
        size = api.cusparseSpMM_bufferSize(h, NT, NT, 1.0, matA, matB, 0.0, matC, cs.CUDA_R_32F)
        buf = torch.empty(max(size, 16), dtype=torch.uint8, device=DEV)
        api.cusparseSpMM_preprocess(h, NT, NT, 1.0, matA, matB, 0.0, matC, cs.CUDA_R_32F, 0, buf)
        fn, a1, b0 = api.real.cusparseSpMM, C.c_float(1.0), C.c_float(0.0)

        def closed():
            api.cusparseSetStream(h, torch.cuda.current_stream().cuda_stream)
            st = fn(h, NT, NT, C.byref(a1), matA, matB, C.byref(b0), matC, cs.CUDA_R_32F, 0, C.c_void_p(buf.data_ptr()))
            assert st == 0, st
        out["closed_us"] = graph_time(closed, calls, reps, warmup)
        gotc = Cc.view(m, n) if order == ROW else Cc.view(n, m).t()
        out["closed_err"] = float((gotc.double() - ref).abs().max())
    except (cs.CuSparseError, AssertionError) as e:
        out["closed_us"], out["closed_err"] = None, f"rejected: {e}"
    finally:
        api.cusparseDestroySpMat(matA)
        api.cusparseDestroyDnMat(matB)
        api.cusparseDestroyDnMat(matC)
        api.cusparseDestroy(h)
    live = int((ci >= 0).sum())
    flops = 2.0 * live * bs * bs * n
    nbytes = ci.numel() * 4 + vals.numel() * vals.element_size() + B.numel() * B.element_size() + m * n * Co.element_size()
    t_flop, t_byte = flops / PEAK_FLOPS, nbytes / PEAK_BYTES
    out.update(kind=name, m=m, bs=bs, density=density, n=n, blocks=live, flops=flops, bytes=nbytes,
               bound="compute" if t_flop >= t_byte else "memory", bound_us=max(t_flop, t_byte) * 1e6,
               ours_tflops=flops / out["ours_us"] / 1e6, ours_gbs=nbytes / out["ours_us"] / 1e3)
    if out["closed_us"]:
        out["closed_tflops"] = flops / out["closed_us"] / 1e6
        out["speedup"] = out["closed_us"] / out["ours_us"]
    del ci, vals, B, Bs, Co, Cc, ref
    torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--quick", action="store_true", help="M = K = 2048, one case per kind: a rehearsal, not a measurement")
    ap.add_argument("--calls", type=int, default=20)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--small", action="store_true", help="the size ladder below the table: where launch cost decides, fp16 column-major")
    ap.add_argument("--native-classes", action="store_true",
                    help="M = K = 64, bs 2 .. 64, every type combination and order, N 8 and 128: the classes the route keeps native")
    ap.add_argument("--structures", action="store_true",
                    help="the closed library's error against fp64 on -1-slot layouts (512 x 512, bs 16, N 72, fp16 -> fp32, column-major)")
    ap.add_argument("--json", default="")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "bell_bench.py measures on the GPU; there is nothing to measure without one"
    m = k = 2048 if a.quick else 16384
    cases = [(bs, d, n, kind) for bs in (16, 32, 64) for d in (0.1, 0.3) for n in (128, 512) for kind in KINDS]
    cases.append((4, 0.1, 128, KINDS[0]))
    if a.quick:
        cases = [(16, 0.1, 128, kd) for kd in KINDS] + [(4, 0.1, 128, KINDS[0])]
    if a.small:                               # (M = K, bs, N): the spmm_blockedell sample's shape, then M = K = 64 .. 4096
        cases = [(4, 2, 3)] + [(mk, bs, nn) for mk in (64, 256, 1024, 2048, 4096) for bs in (2, 16, 64) for nn in (8, 128) if mk >= 2 * bs]
        cases = [(mk, bs, 0.5, nn, KINDS[0]) for mk, bs, nn in cases]
    elif a.native_classes:
        cases = [(64, bs, 0.5, nn, kd) for bs in (2, 16, 32, 64) for kd in KINDS + MORE_KINDS for nn in (8, 128)]
    else:
        cases = [(m, bs, d, n, kd) for bs, d, n, kd in cases]
    res = {"card": card(), "cases": []}
    print(f"# {res['card']}")
    if a.structures:
        kind = ("f16-f32-col", torch.float16, torch.float32, COL)
        print("| structure | ours max err | closed max err |")
        print("|---|---|---|")
        for name, ci in structures(32, 8, 3).items():
            r = run_case(512, 512, 16, None, 72, kind, 2, 1, 1, ci=ci)
            r["structure"] = name
            res["cases"].append(r)
            ce = r["closed_err"] if isinstance(r["closed_err"], str) else f"{r['closed_err']:.3g}"
            print(f"| {name} | {r['ours_err']:.3g} | {ce} |", flush=True)
        cases = []
    print("| kind | M = K | bs | density | N | ours us | closed us | speedup | ours TFLOP/s | ours GB/s | bound (us) | ours err | closed err |")
    print("|---|---|---|---|---|---|---|---|---|---|---|---|---|")
    for mk, bs, d, n, kind in cases:
        r = run_case(mk, mk, bs, d, n, kind, a.calls, a.reps, a.warmup)
        res["cases"].append(r)
        cl = f"{r['closed_us']:.1f}" if r["closed_us"] else "rejected"
        sp = f"{r['speedup']:.2f}x" if r.get("speedup") else "-"
        ce = f"{r['closed_err']:.3g}" if isinstance(r["closed_err"], float) else r["closed_err"][:40]
        print(f"| {r['kind']} | {mk} | {bs} | {d} | {n} | {r['ours_us']:.1f} | {cl} | {sp} | {r['ours_tflops']:.0f} | {r['ours_gbs']:.0f} | "
              f"{r['bound']} ({r['bound_us']:.1f}) | {r['ours_err']:.3g} | {ce} |", flush=True)
    if a.json:
        os.makedirs(os.path.dirname(os.path.abspath(a.json)), exist_ok=True)
        with open(a.json, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
