#!/usr/bin/env python
"""Per-tile timing of the CSR kernels (needs a -DB200_CSR_TRACE build: scripts/trace_tiles.py build|run)."""
import ctypes as C
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
VDIR = os.path.join(ROOT, "cudalibrarysamples_b200", "build", "variants")
TAGS = {"trace_tile": ["-DB200_CSR_TRACE", "-DB200_CSR_KERNEL=0", "-DB200_CSR_MIN_CTAS=5"],
        "trace_pipe": ["-DB200_CSR_TRACE", "-DB200_CSR_KERNEL=1", "-DB200_CSR_MIN_CTAS=4"],
        "trace_pipe3": ["-DB200_CSR_TRACE", "-DB200_CSR_KERNEL=1", "-DB200_CSR_MIN_CTAS=3"]}

if sys.argv[1] == "build":
    from cudalibrarysamples_b200 import build as b
    os.makedirs(VDIR, exist_ok=True)
    for tag, fl in TAGS.items():
        print(b.build_native(extra_flags=fl, out_path=os.path.join(VDIR, f"libb200spmv_{tag}.so"), tag="v_" + tag))
    sys.exit(0)

import numpy as np
import torch
from cudalibrarysamples_b200 import cusparse_api as cs
from cudalibrarysamples_b200 import workloads as W
sys.path.insert(0, os.path.join(ROOT, "scripts"))
from sweep import make_workload

out = {}
for wl in sys.argv[2:] or ["rmat1m"]:
    rows, off, col, val = make_workload(wl)
    x = W.uniform(44, rows)
    for tag in TAGS:
        path = os.path.join(VDIR, f"libb200spmv_{tag}.so")
        api = cs.Api("b200", lib_path=path)
        op = cs.SpMVOperator(api, "csr", rows, rows, dict(off=off, col=col, val=val))
        ntiles = api.lib.b200spmv_csr_num_tiles(rows, col.numel())
        y = torch.zeros(rows, dtype=torch.float64, device="cuda")
        for _ in range(3):
            op(x, y)
        trace = torch.zeros(ntiles * 4, dtype=torch.int64, device="cuda")
        # only -DB200_CSR_TRACE builds define this hook, so no header declares it: the pointer goes as an explicit c_void_p
        api.lib.b200spmv_debug_set_trace(C.c_void_p(trace.data_ptr()))
        op(x, y)
        torch.cuda.synchronize()
        api.lib.b200spmv_debug_set_trace(C.c_void_p(0))
        t = trace.cpu().numpy().reshape(-1, 4)
        o = api.lib.b200spmv_csr_plan_tiles_offset()
        tiles = op.buffer[o:o + (ntiles + 1) * 8].view(torch.int32).view(-1, 2).cpu().numpy().astype(np.int64)
        trows = np.diff(tiles[:, 0]); tnnz = np.diff(tiles[:, 1])
        d1 = t[:, 1] - t[:, 0]; d2 = t[:, 2] - t[:, 1]; dt = t[:, 2] - t[:, 0]
        print(f"== {wl} {tag}: tiles={ntiles}")
        print("   cycles/tile   phase1 mean %.0f p50 %.0f p90 %.0f | phase2 mean %.0f p50 %.0f p90 %.0f | total mean %.0f" % (
            d1.mean(), np.median(d1), np.percentile(d1, 90), d2.mean(), np.median(d2), np.percentile(d2, 90), dt.mean()))
        # by tile class: rows per tile
        for lo, hi in [(0, 16), (16, 64), (64, 256), (256, 768), (768, 4096)]:
            m = (trows >= lo) & (trows < hi)
            if m.any():
                print(f"   rows/tile in [{lo},{hi}): n={m.sum():5d} nnz/tile {tnnz[m].mean():7.0f}  phase1 {d1[m].mean():7.0f}  phase2 {d2[m].mean():7.0f}")
        # per-SM busy span
        sm = t[:, 3]
        spans = []
        for s_ in np.unique(sm):
            mm = sm == s_
            spans.append((t[mm, 2].max() - t[mm, 0].min(), mm.sum(), dt[mm].sum()))
        spans = np.array(spans)
        print("   per-SM: span cycles mean %.0f max %.0f min %.0f | tiles/SM mean %.1f max %d min %d | sum(tile cycles)/span mean %.2f" % (
            spans[:, 0].mean(), spans[:, 0].max(), spans[:, 0].min(), spans[:, 1].mean(), spans[:, 1].max(), spans[:, 1].min(),
            (spans[:, 2] / spans[:, 0]).mean()))
        out[f"{wl}/{tag}"] = dict(phase1=float(d1.mean()), phase2=float(d2.mean()), total=float(dt.mean()))
        op.close()
json.dump(out, open(os.path.join(ROOT, "gpurun_out", "trace_tiles.json"), "w"), indent=1)
