#!/usr/bin/env python
"""Unpreconditioned fp64 BiCGStab (bicgstab_example.c:212-351 with M = I) on the sample's advection-diffusion operator
(workloads.stencil5_csr(grid, mass=0.3, ux=0.3, uy=0.2), b = 0.75 * A * 1, x0 = 0), row-sharded over N GPUs.

  solve  grid 700, tol 1e-10: time to solution
  rate   grid 8192, 200 fixed iterations (tol None): iterations/s

Variants: the fused solver with our SpMV, the fused solver with the closed library's SpMV (a cs.Api("cusparse") operator
inside the same loop), and the torch-op loop with our SpMV.  Times are CUDA events after a warm-up run, the median of
--windows runs, the maximum over ranks.  The card name and power limit are read in the same run.  Bytes per iteration are
computed from the shapes: 2 SpMVs (values, column indices, offsets, x gathered once, y written) plus the BLAS-1 passes.

  python scripts/bicgstab_bench.py [--windows 5] [--chunks 4,8,16,32]
  python -m torch.distributed.run --nproc-per-node N scripts/bicgstab_bench.py --gpus N
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch
import torch.distributed as dist

from cudalibrarysamples_b200 import cusparse_api as cs
from cudalibrarysamples_b200 import workloads as W
from cudalibrarysamples_b200.bicgstab import BicgstabSolver, FusedBicgstabSolver
from cudalibrarysamples_b200.sharded import ShardedCsr

sys.stdout.flush()
_REAL_STDOUT = os.fdopen(os.dup(1), "w")
os.dup2(2, 1)   # only our JSON lines go to the real stdout
ap = argparse.ArgumentParser()
ap.add_argument("--gpus", type=int, default=1)
ap.add_argument("--windows", type=int, default=5)
ap.add_argument("--solve-grid", type=int, default=700)
ap.add_argument("--rate-grid", type=int, default=8192)
ap.add_argument("--iters", type=int, default=200)
ap.add_argument("--chunks", default="", help="also time the fused solver at these graph chunk lengths (one GPU)")
a = ap.parse_args()
world = int(os.environ.get("WORLD_SIZE", "1"))
rank = int(os.environ.get("RANK", "0"))
local = int(os.environ.get("LOCAL_RANK", "0"))
assert world == a.gpus
torch.cuda.set_device(local)
if world > 1:
    dist.init_process_group("nccl", device_id=torch.device("cuda", local))


def card():
    q = subprocess.run(["nvidia-smi", "-i", str(local), "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip() or torch.cuda.get_device_name(local)


def bicgstab_loop_passes():
    """BLAS-1 whole-vector passes per iteration of the sample's loop with M = I (P_aux = P, S_aux = S, so the solves and
    their memsets drop out), counted call by call from bicgstab_example.c:224-347: dots R0.R, R0.V, T.S, T.T; nrm2 of S and
    R; axpys on P (2), X (2), S and R; one scal of P; copies S = R and R = S.  Costs in whole-vector passes: dot 2, nrm2 1,
    axpy 3, scal 2, copy 2.  Returns (passes, host round trips: the 4 dots and 2 norms)."""
    loop = dict(dot=4, nrm2=2, axpy=6, scal=1, copy=2)
    cost = dict(dot=2, nrm2=1, axpy=3, scal=2, copy=2)
    return sum(loop[k] * cost[k] for k in loop), loop["dot"] + loop["nrm2"]


FUSED_PASSES = 2 + 3 + 2 + 7 + 4                           # b200cg_dot, update_s, dot2, update_xr, update_p
# bicgstab(): s = r - alpha v 3, dots r0.v, s.s, t.s, t.t 2 each, x += alpha p 3 and += omega s 3, r = s - omega t 3,
# dots r0.r and r.r 2 each, p -= omega v 3, p *= beta 2, p += r 3
TORCH_PASSES = 3 + 8 + 6 + 3 + 4 + 3 + 2 + 3


def bytes_per_iteration(rows, nnz, passes):
    spmv = nnz * (8 + 4) + (rows + 1) * 4 + rows * 8 + rows * 8     # values + columns, offsets, x once, y written
    return 2 * spmv + passes * rows * 8


def build(grid, impl):
    off, col, val = W.stencil5_csr(grid, mass=0.3, ux=0.3, uy=0.2)
    api = cs.Api(impl)

    def make_local(r, c, arrays, api=api):
        return cs.SpMVOperator(api, "csr", r, c, arrays, preprocess=True)
    sh = ShardedCsr(off, col, val, rank, world, make_local, balance="rows")
    ones = torch.ones(grid * grid, dtype=torch.float64, device="cuda")
    b = sh.new_y_shard()
    sh.spmv(sh.new_x_shard(ones), b, alpha=0.75, beta=0.0)
    return sh, b, int(off[-1].item())


def timed(fn):
    if world > 1:
        dist.barrier()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    res = fn()
    e1.record()
    torch.cuda.synchronize()
    ms = torch.tensor([e0.elapsed_time(e1)], dtype=torch.float64, device="cuda")
    if world > 1:
        dist.all_reduce(ms, op=dist.ReduceOp.MAX)
    return float(ms.item()), res


def true_residual(sh, b, x):
    r = b.clone()
    sh.spmv(x, r, alpha=-1.0, beta=1.0)
    rr = torch.dot(r, r).reshape(1)
    bb = torch.dot(b, b).reshape(1)
    if world > 1:
        dist.all_reduce(rr)
        dist.all_reduce(bb)
    return float(rr.sqrt().item()) / float(bb.sqrt().item())


def measure(solver, max_iters, tol, sh, b):
    solver.run(max_iters, tol)                               # warm-up: modules, plans, graph capture
    times, res = [], None
    for _ in range(a.windows):
        ms, res = timed(lambda: solver.run(max_iters, tol))
        times.append(ms)
    return dict(ms=round(statistics.median(times), 3), ms_all=[round(t, 3) for t in times], status=res.status,
                iterations=res.iterations, rel_true_residual=true_residual(sh, b, res.x))


VARIANTS = [("fused_ours", "b200", FusedBicgstabSolver), ("fused_closed_spmv", "cusparse", FusedBicgstabSolver),
            ("torch_ops_ours", "b200", BicgstabSolver)]
out = dict(card=card(), n_gpus=world, solve={}, rate={})
for case, grid, max_iters, tol in (("solve", a.solve_grid, 5000, 1e-10), ("rate", a.rate_grid, a.iters, None)):
    for name, impl, cls in VARIANTS:
        sh, b, nnz = build(grid, impl)
        m = measure(cls(sh, b), max_iters, tol, sh, b)
        passes = FUSED_PASSES if cls is FusedBicgstabSolver else TORCH_PASSES
        m["bytes_per_iteration_per_rank"] = bytes_per_iteration(sh.rows, sh.nnz, passes)
        if case == "rate":
            m["iters_per_s"] = round(m["iterations"] / (m["ms"] * 1e-3), 2)
            m["GB_per_s_per_rank"] = round(m["bytes_per_iteration_per_rank"] * m["iters_per_s"] / 1e9, 1)
        out[case][name] = m
        sh.local_op.close()
        del sh, b
        torch.cuda.empty_cache()
    if case == "rate" and a.chunks and world == 1:
        sh, b, nnz = build(grid, "b200")
        sweep = {}
        default = FusedBicgstabSolver.CHUNK
        for c in (int(v) for v in a.chunks.split(",")):
            FusedBicgstabSolver.CHUNK = c
            sweep[c] = measure(FusedBicgstabSolver(sh, b), max_iters, tol, sh, b)["ms"]
        FusedBicgstabSolver.CHUNK = default
        out["chunk_sweep_rate_ms"] = sweep
        sh2, b2, _ = build(a.solve_grid, "b200")
        sweep = {}
        for c in (int(v) for v in a.chunks.split(",")):
            FusedBicgstabSolver.CHUNK = c
            sweep[c] = measure(FusedBicgstabSolver(sh2, b2), 5000, 1e-10, sh2, b2)["ms"]
        FusedBicgstabSolver.CHUNK = default
        out["chunk_sweep_solve_ms"] = sweep
        sh.local_op.close()
        sh2.local_op.close()
passes, trips = bicgstab_loop_passes()
out["passes_per_iteration"] = dict(fused=FUSED_PASSES, torch_ops=TORCH_PASSES, sample_loop_m_eq_i=passes, sample_host_round_trips=trips)
if rank == 0:
    print(json.dumps(out), file=_REAL_STDOUT, flush=True)
if world > 1:
    dist.barrier()
    dist.destroy_process_group()
