"""Row-sharded conjugate gradient around the SpMV path (BASELINE.json config 4: 5-pt Poisson 8192^2, fp64, 200 fixed
iterations, iterations/s at 1..8 GPUs).

Restates the loop of the reference's gpu_CG (cuSPARSE/cg/cg_example.c:132-307) without the IC(0) preconditioner: the
reference's preconditioner is a global incomplete Cholesky + two SpSV solves, which does not row-shard (SURVEY.md 8e),
so the sharded driver is plain CG (the SpMV call per iteration, cg_example.c:220-224, is the part this project
replaces).  Same set-up as the sample: b = 0.75 * A * 1, x0 = 0 (cg_example.c:405-420).

Host logic only: the local SpMV is injected, so the gloo tests drive it with the CPU oracle and cg_bench.py with the
sm_90a operator.  Vector updates and dot products are torch ops (plumbing); the dots are all-reduced over ranks.
"""
from __future__ import annotations

import contextlib

import torch
import torch.distributed as dist

from .sharded import ShardedCsr


@contextlib.contextmanager
def side_stream(sh: ShardedCsr):
    """A fresh stream for CUDA-graph capture (capture needs a stream other than the default one), made current, with the
    library handles of the sharded operator moved onto it; on exit the handles go back and the caller's stream waits for it."""
    main = torch.cuda.current_stream()
    side = torch.cuda.Stream()
    side.wait_stream(main)
    ops = [op for op in (getattr(sh, "local_op", None), getattr(sh, "own_op", None)) if op is not None and hasattr(op, "handle")]
    try:
        with torch.cuda.stream(side):
            for op in ops:
                op.api.cusparseSetStream(op.handle, side.cuda_stream)
            yield side
    finally:
        main.wait_stream(side)
        for op in ops:
            op.api.cusparseSetStream(op.handle, main.cuda_stream)


def _dot(a: torch.Tensor, b: torch.Tensor, world: int, group=None) -> torch.Tensor:
    d = torch.dot(a, b).reshape(1)
    if world > 1:
        dist.all_reduce(d, group=group)
    return d


def conjugate_gradient(sh: ShardedCsr, b_shard: torch.Tensor, iters: int, x0_shard: torch.Tensor | None = None,
                       tol: float | None = None):
    """Plain CG on this rank's row block; requires the x / y distributions of `sh` to coincide (equal row blocks), which
    is the case for the stencil matrices of config 4 when rows % world == 0.

    Returns (x_shard, residual_norms) -- residual_norms[k] = ||r_k||_2 (global), k = 0 .. iters_done.
    """
    assert sh.rows == sh.x_block or sh.world == 1, "CG needs y-rows == x-block (regular matrix, rows % world == 0)"
    world, group = sh.world, sh.group
    x = torch.zeros_like(b_shard) if x0_shard is None else x0_shard.clone()
    r = b_shard.clone()
    t = torch.zeros_like(b_shard)
    if x0_shard is not None:
        sh.spmv(x, r, alpha=-1.0, beta=1.0)            # r = b - A x0   (cg_example.c:153-160)
    p = r.clone()
    delta = _dot(r, r, world, group)
    norms = [delta.sqrt()]
    for _ in range(iters):
        sh.spmv(p, t, alpha=1.0, beta=0.0)             # T = A * P      (cg_example.c:220-224)
        denom = _dot(t, p, world, group)
        alpha = delta / denom                          # 1-element device tensors: no host sync in the loop
        x.addcmul_(p, alpha)                           # X += alpha P   (cg_example.c:236-239), one pass, no temporary
        r.addcmul_(t, alpha, value=-1.0)               # R -= alpha T   (cg_example.c:241-244)
        delta_new = _dot(r, r, world, group)
        norms.append(delta_new.sqrt())
        if tol is not None and float(norms[-1]) < tol * float(norms[0]):
            break
        beta = delta_new / delta
        torch.addcmul(r, p, beta, out=p)               # P = beta P + R (cg_example.c:280-286), one pass
        delta = delta_new
    return x, torch.cat(norms)


class CgSolver:
    """conjugate_gradient() packaged for repeated timed runs (bench.py's cg_config4 leg, scripts/cg_bench.py): torch ops."""

    def __init__(self, sh: ShardedCsr, b_shard: torch.Tensor):
        self.sh, self.b = sh, b_shard

    def run(self, iters: int):
        x, norms = conjugate_gradient(self.sh, self.b, iters)
        return x, [float(v) for v in norms.tolist()]

    def describe(self) -> str:
        return ("plain CG (cg_example.c:215-287 without the IC(0) preconditioner), SpMV through the C ABI, vector updates as "
                "single-pass torch ops (addcmul), dots all-reduced over ranks, no host synchronisation inside the loop")


class FusedCgSolver:
    """The same iteration on the fused sm_90a BLAS-1 kernels of csrc/cg_fused.cu (b200cg_dot / _update_r / _update_xp): per
    iteration 1 SpMV + 3 kernels, every scalar in device memory, partial dots all-reduced over ranks; on one GPU two
    iterations are captured in a CUDA graph and replayed (graph_capture_example.c:118-135 pattern)."""

    def __init__(self, sh: ShardedCsr, b_shard: torch.Tensor, use_graph: bool | None = None):
        import os
        from . import lib as _lib
        self.L = _lib.shim()
        self.sh, self.b = sh, b_shard
        self.n = int(b_shard.numel())
        dev = b_shard.device
        self.ws = torch.zeros(self.L.b200cg_workspace_bytes(), dtype=torch.uint8, device=dev)
        self.scal = torch.zeros(8, dtype=torch.float64, device=dev)        # [0], [1]: delta of even / odd iterations, [2]: t.p
        self.use_graph = (sh.world == 1 and os.environ.get("B200CG_GRAPH", "1") != "0") if use_graph is None else use_graph
        self.graph_error = None
        # T = A*P and T . P in one kernel where the local matrix allows it (all rows short: csr_short_kernel's DOT variant).
        # Opt-in: the extra live registers of the DOT variant spill in the 48-register kernel, so on 5-pt 8192^2 it is no
        # faster than the plain kernel + b200cg_dot.
        self.fuse_dot = os.environ.get("B200CG_FUSE_DOT", "0") == "1" and hasattr(sh, "can_fuse_dot") and sh.can_fuse_dot()

    def _stream(self):
        return torch.cuda.current_stream().cuda_stream

    def _check(self, rc, what):
        if rc != 0:
            raise RuntimeError(f"{what} failed with code {rc}")

    def _dot(self, a, b, out):
        self._check(self.L.b200cg_dot(self._stream(), self.n, a.data_ptr(), b.data_ptr(), out.data_ptr(), self.ws.data_ptr()), "b200cg_dot")
        if self.sh.world > 1:
            dist.all_reduce(out, group=self.sh.group)

    def _iteration(self, x, r, p, t, cur):
        """one CG iteration; delta_k lives in scal[cur], delta_{k+1} goes to scal[1 - cur]"""
        s = self.scal
        if self.fuse_dot:
            self.sh.spmv_dot(p, t, s[2:3])                                   # T = A * P and denom = T . P in one pass (:220-227)
            if self.sh.world > 1:
                dist.all_reduce(s[2:3], group=self.sh.group)
        else:
            self.sh.spmv(p, t, alpha=1.0, beta=0.0)                          # T = A * P      (cg_example.c:220-224)
            self._dot(t, p, s[2:3])                                          # denom = T . P  (:227)
        nxt = 1 - cur
        # 8 vector passes after the dot's 2: R -= aT with delta' = R.R, then X += aP and P = R + (delta'/delta) P in one pass (P read once)
        self._check(self.L.b200cg_update_r(self._stream(), self.n, r.data_ptr(), t.data_ptr(), s[cur:cur + 1].data_ptr(), s[2:3].data_ptr(),
                                           s[nxt:nxt + 1].data_ptr(), self.ws.data_ptr()), "b200cg_update_r")       # (:241-247)
        if self.sh.world > 1:
            dist.all_reduce(s[nxt:nxt + 1], group=self.sh.group)
        self._check(self.L.b200cg_update_xp(self._stream(), self.n, x.data_ptr(), p.data_ptr(), r.data_ptr(), s[cur:cur + 1].data_ptr(),
                                            s[2:3].data_ptr(), s[nxt:nxt + 1].data_ptr()), "b200cg_update_xp")       # (:236-239, :280-286)

    def run(self, iters: int):
        x = torch.zeros_like(self.b)
        r = self.b.clone()
        # the search direction lives inside the assembled x buffer: no staging copy in front of every product
        own = self.sh.own_x_view() if hasattr(self.sh, "own_x_view") and (self.sh.world == 1 or self.sh.exchange == "halo") else None
        p = own if own is not None and own.numel() == r.numel() and own.data_ptr() % 16 == 0 else torch.empty_like(r)
        p.copy_(r)
        t = torch.zeros_like(self.b)
        self._dot(r, r, self.scal[0:1])
        first = self.scal[0:1].clone()
        done = 0
        if self.use_graph and iters >= 4 and self.graph_error is None:
            try:
                done = self._run_graphed(x, r, p, t, iters)
            except Exception as e:                   # capture refused (driver / library version): plain launches instead
                self.graph_error = repr(e)
                torch.cuda.synchronize()
                x.zero_(); r.copy_(self.b); p.copy_(self.b)
                self._dot(r, r, self.scal[0:1])
                done = 0
        for k in range(done, iters):
            self._iteration(x, r, p, t, k & 1)
        last = self.scal[iters & 1:(iters & 1) + 1]
        norms = torch.cat([first, last]).sqrt()
        return x, [float(v) for v in norms.tolist()]

    def _run_graphed(self, x, r, p, t, iters):
        with side_stream(self.sh) as side:
            self._iteration(x, r, p, t, 0)            # two eager iterations: warm-up of every kernel on this stream
            self._iteration(x, r, p, t, 1)
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g, stream=side):
                self._iteration(x, r, p, t, 0)
                self._iteration(x, r, p, t, 1)
            done = 4                                  # the capture pass does not execute: 2 eager + first replay below = 4
            g.replay()
            while done + 2 <= iters:
                g.replay()
                done += 2
        self._graph = g
        return done

    def describe(self) -> str:
        how = "two iterations captured in a CUDA graph and replayed" if self.use_graph and self.graph_error is None else "plain stream launches"
        spmv = ("T = A*P and T.P in one csr_short_kernel launch (b200spmv_csr_short_mv_dot)" if self.fuse_dot
                else "SpMV through the C ABI + b200cg_dot")
        return ("CG (cg_example.c:215-287 without the IC(0) preconditioner): " + spmv + " + fused sm_90a BLAS-1 kernels "
                "(b200cg_update_r = axpy + nrm2 in one pass, b200cg_update_xp = x and p updates in one pass: 10 vector passes per iteration with the dot), all scalars on the device, "
                + how + (f" (graph capture failed: {self.graph_error})" if self.graph_error else ""))


def make_cg_solver(sh: ShardedCsr, b_shard: torch.Tensor, fused: bool | None = None):
    """The fused driver on CUDA (the product), the torch-op driver on CPU (gloo tests with the oracle as local kernel)."""
    if fused is None:
        fused = b_shard.is_cuda
    return FusedCgSolver(sh, b_shard) if fused else CgSolver(sh, b_shard)
