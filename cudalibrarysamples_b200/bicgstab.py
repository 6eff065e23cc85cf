"""Row-sharded BiCGStab around the SpMV path, for the non-symmetric systems that CG cannot solve.

Restates the loop of the reference's gpu_BiCGStab (cuSPARSE/bicgstab/bicgstab_example.c:212-351) without its ILU(0)
preconditioner (M = I): a global incomplete LU and its two triangular solves do not row-shard, so, as for CG (cg.py), the
sharded solver is the plain method.  Same set-up as the sample: b = 0.75 * A * 1, x0 = 0 (bicgstab_example.c:423-437).

  * `bicgstab`: the loop as torch ops with host-side scalars and decisions (host logic only: the local SpMV is injected, so
    the gloo tests drive it with the CPU oracle); the dots are all-reduced over ranks.
  * `FusedBicgstabSolver`: the same iteration on the fused sm_90a kernels of csrc/bicgstab_fused.cu.  Every scalar and every
    decision stays on the device, so on one GPU a chunk of iterations is captured in a CUDA graph and replayed, and the host
    learns about convergence one chunk late without stopping the GPU.

Both follow one status protocol (include/b200spmv.h, B200BICGSTAB_*): the solve stops converged at s (||s|| < tol ||r0||,
x += alpha p, r = s), converged at r (||r|| < tol ||r0||), or at a breakdown (r0 . v = 0, t . t = 0, omega = 0, r0 . r = 0, a
non-finite scalar) that leaves x as the last finished iteration left it.  tol = None: no convergence test, exactly max_iters
iterations unless a breakdown comes first.
"""
from __future__ import annotations

import contextlib
import ctypes as C
import math
from typing import NamedTuple

import torch
import torch.distributed as dist

from .cg import side_stream
from .sharded import ShardedCsr

RUNNING, CONVERGED_S, CONVERGED_R = 0, 1, 2
BREAKDOWN_DENOM, BREAKDOWN_TT, BREAKDOWN_OMEGA, BREAKDOWN_RHO, BREAKDOWN_NONFINITE = 3, 4, 5, 6, 7
STATUS_NAMES = {RUNNING: "running", CONVERGED_S: "converged_s", CONVERGED_R: "converged_r", BREAKDOWN_DENOM: "breakdown_denom",
                BREAKDOWN_TT: "breakdown_tt", BREAKDOWN_OMEGA: "breakdown_omega", BREAKDOWN_RHO: "breakdown_rho",
                BREAKDOWN_NONFINITE: "breakdown_nonfinite"}
# state slots (doubles) of the fused kernels' state block
RHO, ALPHA, OMEGA, DENOM, S2, TS, TT, RHO_NEW, R2, THRESHOLD = range(10)


class BicgstabResult(NamedTuple):
    x: torch.Tensor              # this rank's block of the solution
    status: str                  # STATUS_NAMES: "running" means max_iters ran out
    iterations: int              # finished iterations (x is the iterate after them)
    history: list                # ||r_k|| for k = 0 .. iterations (||s|| for the last one when converged at s)


def _dots(pairs, world: int, group=None) -> list:
    """the dot products of (a, b) pairs, all-reduced over ranks in one call, as host floats"""
    d = torch.stack([torch.dot(a, b) for a, b in pairs])
    if world > 1:
        dist.all_reduce(d, group=group)
    return [float(v) for v in d.tolist()]


def _finite(*v) -> bool:
    return all(math.isfinite(a) for a in v)


def bicgstab(sh: ShardedCsr, b_shard: torch.Tensor, max_iters: int, tol: float | None = None,
             x0_shard: torch.Tensor | None = None) -> BicgstabResult:
    """Unpreconditioned BiCGStab on this rank's row block, scalars on the host (one round trip per reduction group, as in the
    sample).  Needs the x and y distributions of `sh` to coincide (equal row blocks), like conjugate_gradient."""
    assert sh.rows == sh.x_block or sh.world == 1, "BiCGStab needs y-rows == x-block (regular matrix, rows % world == 0)"
    world, group = sh.world, sh.group
    x = torch.zeros_like(b_shard) if x0_shard is None else x0_shard.clone()
    r0 = b_shard.clone()
    if x0_shard is not None:
        sh.spmv(x, r0, alpha=-1.0, beta=1.0)                   # R0 = b - A X0   (bicgstab_example.c:185-195)
    r, p = r0.clone(), r0.clone()
    v, s, t = torch.zeros_like(r0), torch.zeros_like(r0), torch.zeros_like(r0)
    (rho_new,) = _dots([(r0, r0)], world, group)
    rho = rho_new
    threshold = -1.0 if tol is None else tol * math.sqrt(rho)
    history = [math.sqrt(rho)]
    status = BREAKDOWN_NONFINITE if not _finite(rho) else CONVERGED_R if rho == 0 else RUNNING
    k = 0
    for _ in range(max_iters):
        if status != RUNNING:
            break
        sh.spmv(p, v, alpha=1.0, beta=0.0)                     # V = A P        (:260-265)
        (denom,) = _dots([(r0, v)], world, group)              # r0 . V         (:267-269)
        alpha = rho_new / denom if denom != 0 else math.inf
        if denom == 0:
            status = BREAKDOWN_DENOM
            break
        if not _finite(alpha):
            status = BREAKDOWN_NONFINITE
            break
        torch.add(r, v, alpha=-alpha, out=s)                   # S = R - alpha V (:281-287)
        rho = rho_new
        sh.spmv(s, t, alpha=1.0, beta=0.0)                     # T = A S        (:315-320)
        s2, ts, tt = _dots([(s, s), (t, s), (t, t)], world, group)
        if not _finite(s2):
            status = BREAKDOWN_NONFINITE
            break
        if math.sqrt(s2) < threshold:                          # ||S|| < threshold (:290-293)
            x.add_(p, alpha=alpha)
            r.copy_(s)
            k += 1
            history.append(math.sqrt(s2))
            status = CONVERGED_S
            break
        omega = ts / tt if tt != 0 else math.inf
        if not _finite(ts, tt):
            status = BREAKDOWN_NONFINITE
        elif tt == 0:
            status = BREAKDOWN_TT
        elif not _finite(omega):
            status = BREAKDOWN_NONFINITE
        elif omega == 0:
            status = BREAKDOWN_OMEGA
        if status != RUNNING:
            break
        x.add_(p, alpha=alpha).add_(s, alpha=omega)            # X += alpha P + omega S (:272-275, :330-335)
        torch.add(s, t, alpha=-omega, out=r)                   # R = S - omega T (:338-345)
        rho_new, r2 = _dots([(r0, r), (r, r)], world, group)
        k += 1
        history.append(math.sqrt(r2) if r2 >= 0 else math.nan)
        beta = (rho_new / rho) * (alpha / omega) if rho != 0 and omega != 0 else math.inf
        if not _finite(r2, rho_new):
            status = BREAKDOWN_NONFINITE
        elif math.sqrt(r2) < threshold:                        # ||R|| < threshold (:347-350)
            status = CONVERGED_R
        elif rho_new == 0:
            status = BREAKDOWN_RHO
        elif not _finite(beta):
            status = BREAKDOWN_NONFINITE
        if status != RUNNING:
            break
        p.sub_(v, alpha=omega).mul_(beta).add_(r)              # P = R + beta (P - omega V) (:230-242)
    return BicgstabResult(x, STATUS_NAMES[status], k, history)


class BicgstabSolver:
    """bicgstab() packaged for repeated timed runs (scripts/bicgstab_bench.py): torch ops, host-side scalars."""

    def __init__(self, sh: ShardedCsr, b_shard: torch.Tensor):
        self.sh, self.b = sh, b_shard

    def run(self, max_iters: int, tol: float | None = None, x0_shard: torch.Tensor | None = None) -> BicgstabResult:
        return bicgstab(self.sh, self.b, max_iters, tol, x0_shard)

    def describe(self) -> str:
        return ("unpreconditioned BiCGStab (bicgstab_example.c:212-351 with M = I), SpMV through the C ABI, vector updates as "
                "torch ops, dots all-reduced over ranks, scalars and decisions on the host (3 round trips per iteration)")


class FusedBicgstabSolver:
    """The same iteration on the fused sm_90a kernels of csrc/bicgstab_fused.cu: per iteration 2 SpMVs + b200cg_dot + 4
    kernels (18 whole-vector passes), every scalar and decision in a device-resident state block.

    On one GPU a chunk of CHUNK iterations is captured in a CUDA graph and replayed.  After each chunk the state header is
    copied to pinned host memory asynchronously; the host reads the copy of the chunk before, so it never waits for the
    chunk in flight, and the chunk it overshoots by is harmless: once stopped, the state is frozen.  On several GPUs the
    kernels are plain launches with 3 all-reduces per iteration (denom; s2, ts, tt; rho_new, r2) and the same lagged check,
    which every rank takes at the same chunk because the status comes from all-reduced scalars."""

    CHUNK = 8          # iterations per replay, measured on an H100 (DESIGN.md 3.27)

    def __init__(self, sh: ShardedCsr, b_shard: torch.Tensor, use_graph: bool | None = None):
        from . import lib as _lib
        assert sh.rows == sh.x_block or sh.world == 1, "BiCGStab needs y-rows == x-block (regular matrix, rows % world == 0)"
        self.L = _lib.shim()
        self.sh, self.b = sh, b_shard
        self.n = int(b_shard.numel())
        self.ws = torch.zeros(self.L.b200bicgstab_workspace_bytes(), dtype=torch.uint8, device=b_shard.device)
        self.use_graph = sh.world == 1 if use_graph is None else use_graph
        sb, ib, hb = C.c_int32(), C.c_int32(), C.c_int32()
        self.L.b200bicgstab_state_layout(0, C.byref(sb), C.byref(ib), C.byref(hb))
        self.status_word, self.iter_word, self.header_doubles = sb.value // 4, ib.value // 4, hb.value // 8
        self._graph = None

    def _stream(self):
        return torch.cuda.current_stream().cuda_stream

    def _check(self, rc, what):
        if rc != 0:
            raise RuntimeError(f"{what} failed with code {rc}")

    def _allreduce(self, lo, hi):
        if self.sh.world > 1:
            dist.all_reduce(self.state[lo:hi], group=self.sh.group)

    def _iteration(self):
        L, n, st, ws, sp = self.L, self.n, self.state.data_ptr(), self.ws.data_ptr(), self.state.data_ptr
        x, r, p, v, s, t, r0 = self.x, self.r, self.p, self.v, self.s, self.t, self.r0
        self.sh.spmv(p, v, alpha=1.0, beta=0.0)                                            # V = A P
        self._check(L.b200cg_dot(self._stream(), n, r0.data_ptr(), v.data_ptr(), sp() + 8 * DENOM, ws), "b200cg_dot")
        self._allreduce(DENOM, DENOM + 1)
        self._check(L.b200bicgstab_update_s(self._stream(), n, r.data_ptr(), v.data_ptr(), s.data_ptr(), st, ws), "b200bicgstab_update_s")
        self.sh.spmv(s, t, alpha=1.0, beta=0.0)                                            # T = A S
        self._check(L.b200bicgstab_dot2(self._stream(), n, t.data_ptr(), s.data_ptr(), st, ws), "b200bicgstab_dot2")
        self._allreduce(S2, TT + 1)
        self._check(L.b200bicgstab_update_xr(self._stream(), n, x.data_ptr(), r.data_ptr(), p.data_ptr(), s.data_ptr(), t.data_ptr(),
                                             r0.data_ptr(), st, ws), "b200bicgstab_update_xr")
        self._allreduce(RHO_NEW, R2 + 1)
        self._check(L.b200bicgstab_update_p(self._stream(), n, p.data_ptr(), r.data_ptr(), v.data_ptr(), st), "b200bicgstab_update_p")

    def _status(self, header: torch.Tensor) -> int:
        return int(header.view(torch.int32)[self.status_word])

    def run(self, max_iters: int, tol: float | None = None, x0_shard: torch.Tensor | None = None) -> BicgstabResult:
        L, b = self.L, self.b
        self.x = torch.zeros_like(b) if x0_shard is None else x0_shard.clone()
        self.r0 = b.clone()
        if x0_shard is not None:
            self.sh.spmv(self.x, self.r0, alpha=-1.0, beta=1.0)                            # R0 = b - A X0
        self.r, self.p, self.v, self.s, self.t = (torch.empty_like(b) for _ in range(5))
        hist = max_iters + 1
        self.state = torch.zeros(L.b200bicgstab_state_layout(hist, None, None, None) // 8, dtype=torch.float64, device=b.device)
        self._check(L.b200cg_dot(self._stream(), self.n, self.r0.data_ptr(), self.r0.data_ptr(), self.state.data_ptr() + 8 * RHO_NEW,
                                 self.ws.data_ptr()), "b200cg_dot")
        self._allreduce(RHO_NEW, RHO_NEW + 1)
        self._check(L.b200bicgstab_init(self._stream(), self.n, self.r0.data_ptr(), self.r.data_ptr(), self.p.data_ptr(),
                                        self.state.data_ptr(), hist, -1.0 if tol is None else float(tol)), "b200bicgstab_init")
        header = self.state[:self.header_doubles]
        host = [torch.empty(self.header_doubles, dtype=torch.float64, pin_memory=True) for _ in range(2)]
        events = [torch.cuda.Event(), torch.cuda.Event()]
        self._graph = None
        done, c = 0, 0
        with side_stream(self.sh) if self.use_graph else contextlib.nullcontext() as side:
            while done < max_iters:
                k = min(self.CHUNK, max_iters - done)
                if self._graph is not None and k == self.CHUNK:
                    self._graph.replay()
                else:
                    for _ in range(k):
                        self._iteration()
                done += k
                host[c & 1].copy_(header, non_blocking=True)
                events[c & 1].record()
                if self.use_graph and self._graph is None and done < max_iters:
                    # every kernel has run once on this stream: capture one chunk (capture does not execute it)
                    g = torch.cuda.CUDAGraph()
                    with torch.cuda.graph(g, stream=side):
                        for _ in range(self.CHUNK):
                            self._iteration()
                    self._graph = g
                if c >= 1:
                    events[(c - 1) & 1].synchronize()
                    if self._status(host[(c - 1) & 1]) != RUNNING:
                        break
                c += 1
        torch.cuda.current_stream().synchronize()
        head = header.cpu()
        status, iters = self._status(head), int(head.view(torch.int32)[self.iter_word])
        history = self.state[self.header_doubles:self.header_doubles + iters + 1].tolist()
        return BicgstabResult(self.x, STATUS_NAMES[status], iters, history)

    def replay(self, times: int = 1):
        """Replays the captured chunk again (after run()): once the solve has stopped this changes nothing."""
        with side_stream(self.sh):
            for _ in range(times):
                self._graph.replay()

    def describe(self) -> str:
        how = f"{self.CHUNK} iterations captured in a CUDA graph and replayed" if self.use_graph else "plain stream launches"
        return ("unpreconditioned BiCGStab (bicgstab_example.c:212-351 with M = I): 2 SpMVs through the C ABI + b200cg_dot + fused "
                "sm_90a kernels (b200bicgstab_update_s / _dot2 / _update_xr / _update_p: 18 vector passes per iteration), "
                "scalars, convergence and breakdown decided on the device, " + how)


def make_bicgstab_solver(sh: ShardedCsr, b_shard: torch.Tensor, fused: bool | None = None):
    """The fused driver on CUDA (the product), the torch-op driver on CPU (gloo tests with the oracle as local kernel)."""
    if fused is None:
        fused = b_shard.is_cuda
    return FusedBicgstabSolver(sh, b_shard) if fused else BicgstabSolver(sh, b_shard)
