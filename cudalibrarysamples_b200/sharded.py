"""Row-block sharding of a square CSR matrix over the GPUs of one box (one process per GPU, torch.distributed).

SpMV shards naturally by contiguous row blocks (SURVEY.md 8e): rank g owns rows [R_g, R_{g+1}) of A -- chosen so every
rank holds ~nnz/G non-zeros, not rows/G, because R-MAT rows are skewed -- plus the matching slice of y.  x is distributed in
EQUAL blocks (not by the row blocks), so the exchange moves exactly |x|*(G-1)/G bytes per rank, no padding, and the
assembled buffer is x: the local product is an ordinary rows_g x cols CSR SpMV through the same C ABI as the single-GPU
path, on the caller's unmodified column indices.

The exchange of x is the path's only communication step, and with a plain all-gather in front of the kernel it is fully
exposed.  So the local matrix is split ONCE at set-up into two column panels:

    own panel     columns of this rank's own x block  -> needs nothing from the other ranks
    remote panel  all other columns                   -> needs the assembled x

and a step is:  start the exchange  ||  y = alpha*A_own*x_own + beta*y   ->   wait   ->   y += alpha*A_remote*x.
Exchange mechanisms (chosen at set-up, structure-only, like the kernels' plans):

    "p2p"        x shards live in symmetric memory (torch.distributed._symmetric_memory: CUDA IPC / fabric handles mapped
                 into every rank); one device-side barrier (csrc/peer_sync.cu: flags in peer memory, epoch on the device), then every rank PULLS the other shards with copy-engine
                 peer copies over NVLink (no SMs, no NCCL kernels) on side streams, starting with a different peer on every
                 rank so no source is read by two ranks at once.  Double-buffered shards: one barrier per step suffices.
    "allgather"  one NCCL all_gather_into_tensor on a side stream (fallback when symmetric memory is unavailable)
    "halo"       banded matrices: only the needed column ranges are sent (5-pt Poisson 8192^2 on 8 GPUs: 2 x 64 KB per rank)

Host logic only -- the local kernel is injected (`make_local_op`) so the world_size-2 gloo tests on CPU can drive the
same code with the CPU oracle, while bench.py passes the sm_90a operator.
"""
from __future__ import annotations

import ctypes as C
import os
from typing import Callable

import torch
import torch.distributed as dist


def split_rows_by_nnz(off: torch.Tensor, world: int, row_weight: float = 0.0) -> torch.Tensor:
    """Row boundaries R_0=0 <= ... <= R_world=rows with ~equal WORK per block (prefix search on rowOff).

    work(rows [a, b)) = non-zeros + row_weight * rows: a row costs the kernels something even when it is short or empty
    (its y entry, its end-of-row reduction), so on skewed matrices a block of many light rows is slower than a block of few
    heavy rows with the same non-zeros (R-MAT at N = 2 splits into a block of many light rows and one of few heavy rows).  row_weight = 0
    is the plain nnz balance of SURVEY.md 8(e); the merge-path view (items = rows + nnz) is row_weight = 1."""
    rows = off.numel() - 1
    o = off.to(torch.int64) - off[0].to(torch.int64)
    if row_weight:
        o = o + (torch.arange(rows + 1, dtype=torch.float64, device=off.device) * row_weight).to(torch.int64)
    nnz = int(o[-1].item())
    targets = torch.tensor([(nnz * g) // world for g in range(1, world)], dtype=torch.int64, device=off.device)
    inner = torch.searchsorted(o.contiguous(), targets, right=False).clamp_(0, rows)
    b = torch.cat([torch.zeros(1, dtype=torch.int64, device=off.device), inner,
                   torch.full((1,), rows, dtype=torch.int64, device=off.device)])
    return torch.cummax(b, 0).values


def split_column_panels(off: torch.Tensor, col: torch.Tensor, val: torch.Tensor, lo: int, hi: int):
    """(off, col, val) of the sub-matrices with columns inside / outside [lo, hi); row order and column order are kept."""
    own = (col >= lo) & (col < hi)
    cs = torch.zeros(col.numel() + 1, dtype=torch.int64, device=col.device)
    cs[1:] = torch.cumsum(own.to(torch.int64), 0)
    o64 = off.to(torch.int64) - off[0].to(torch.int64)
    inside = cs[o64]
    off_own = inside.to(torch.int32).contiguous()
    off_rem = (o64 - inside).to(torch.int32).contiguous()
    rem = ~own
    return (off_own, col[own].contiguous(), val[own].contiguous()), (off_rem, col[rem].contiguous(), val[rem].contiguous())


def split_column_groups(off: torch.Tensor, col: torch.Tensor, val: torch.Tensor, blk: int, groups):
    """One CSR per group of x blocks: groups = [[b0, b1, ...], ...] (block ids, every block in exactly one group); the g-th
    result holds the entries whose column block  col // blk  belongs to groups[g].  Row and column order are kept."""
    nblocks = sum(len(g) for g in groups)
    owner = torch.empty(nblocks, dtype=torch.int64, device=col.device)
    for gi, g in enumerate(groups):
        for b in g:
            owner[b] = gi
    gid = owner[torch.div(col.to(torch.int64), blk, rounding_mode="floor")]
    o64 = off.to(torch.int64) - off[0].to(torch.int64)
    out = []
    for gi in range(len(groups)):
        sel = gid == gi
        cs = torch.zeros(col.numel() + 1, dtype=torch.int64, device=col.device)
        cs[1:] = torch.cumsum(sel.to(torch.int64), 0)
        out.append((cs[o64].to(torch.int32).contiguous(), col[sel].contiguous(), val[sel].contiguous()))
    return out


class ShardedCsr:
    """This rank's row block of a global square CSR matrix plus the exchange plan for x.

    Two distributions, both fixed at set-up:
      * A and y by contiguous row blocks with ~nnz/G non-zeros each (rows [r0, r1) on this rank);
      * x by EQUAL blocks of x_block = ceil(n/G) entries (the last one zero-padded), so the assembled vector is x itself:
        column indices need no remapping.
    (In a solver loop y becomes the next x: with skewed matrices the two distributions differ and the hand-over is a
    redistribution of the row-block / equal-block overlap; for banded matrices they coincide up to a halo.)
    """

    def __init__(self, off: torch.Tensor, col: torch.Tensor, val: torch.Tensor, rank: int, world: int,
                 make_local_op: Callable[[int, int, dict], Callable], group=None, base: int = 0, balance: str = "nnz",
                 exchange: str = "auto", overlap: bool = True, row_weight: float = 0.0):
        assert base == 0
        self.rank, self.world, self.group = rank, world, group
        n = off.numel() - 1
        self.global_rows = n
        self.global_nnz = int(off[-1].item())
        if balance == "nnz":
            self.bounds = split_rows_by_nnz(off, world, row_weight)   # [world+1], identical on every rank
        else:   # "rows": equal row blocks == the x blocks (regular matrices; lets a solver hand y over as the next x)
            blk = max(1, (n + world - 1) // world)
            self.bounds = torch.tensor([min(g * blk, n) for g in range(world + 1)], dtype=torch.int64, device=off.device)
        b = self.bounds.tolist()
        self.r0, self.r1 = b[rank], b[rank + 1]
        self.rows = self.r1 - self.r0
        self.x_block = max(1, (n + world - 1) // world)
        self.pad = self.x_block                                    # length of one x shard
        n0, n1 = int(off[self.r0].item()), int(off[self.r1].item())
        self.off = (off[self.r0:self.r1 + 1].to(torch.int64) - n0).to(torch.int32).contiguous()
        self.col = col[n0:n1].contiguous()
        self.val = val[n0:n1].contiguous()
        self.nnz = n1 - n0
        self.cols_padded = world * self.x_block
        self.x_full = torch.zeros(self.cols_padded, dtype=val.dtype, device=val.device)
        self._step = 0
        self._plan_exchange(exchange)
        # Column panels: only where the whole x is exchanged AND the exchange is long enough to be worth hiding.  The split
        # slows the local product (two plans, y read back for the second panel, shorter rows), which the short exchange of
        # 2 GPUs does not pay back; from 4 GPUs on (>= 24 MB received per rank) the hidden exchange is worth it.
        min_world = int(os.environ.get("B200SPMV_PANELS_FROM", "4"))
        self.panels = overlap and world >= min_world and self.exchange in ("allgather", "p2p") and self.rows > 0
        # blocks in the order they arrive (staggered: rank r pulls r+1, r+2, ... so that no source is read twice at once)
        self.pull_order = [(rank + 1 + i) % world for i in range(world - 1)]
        if self.panels:
            # own block first, then the remote blocks in arrival order, in at most 3 groups (larger groups last: the later
            # a group, the more of the exchange is already behind it)
            ng = min(world - 1, int(os.environ.get("B200SPMV_REMOTE_GROUPS", "3")))
            base, extra = divmod(world - 1, ng)
            sizes = [base + (1 if i >= ng - extra else 0) for i in range(ng)]
            self.panel_groups, k = [[rank]], 0
            for sz in sizes:
                self.panel_groups.append(self.pull_order[k:k + sz])
                k += sz
            parts = split_column_groups(self.off, self.col, self.val, self.x_block, self.panel_groups)
            self.panel_nnz = [int(c.numel()) for (_, c, _) in parts]
            self.own_nnz, self.remote_nnz = self.panel_nnz[0], sum(self.panel_nnz[1:])
            self.panel_ops = [make_local_op(self.rows, self.cols_padded, dict(off=o, col=c, val=v, role="own" if gi == 0 else "remote"))
                              for gi, (o, c, v) in enumerate(parts)]
            self.own_op, self.remote_op = self.panel_ops[0], self.panel_ops[-1]
            self.local_op = self.panel_ops[-1]        # (kept for callers that close "the" local operator)
        else:
            self.local_op = make_local_op(self.rows, self.cols_padded, dict(off=self.off, col=self.col, val=self.val, role="whole"))
        if self.exchange == "p2p":
            self._init_p2p()
        elif self.exchange == "allgather" and val.is_cuda and world > 1:
            self.side = torch.cuda.Stream()
            self.ev_in, self.ev_out = torch.cuda.Event(), torch.cuda.Event()

    # ------------------------------------------------------------------------------------------------ planning
    def _plan_exchange(self, exchange: str):
        """Structure-only preprocessing of the exchange step: which part of x does this row block actually read?

        The local columns span [cmin, cmax].  For a banded matrix that is this rank's own block plus a halo (5-pt
        Poisson 8192^2 on 8 GPUs: 2 x 64 KB instead of 470 MB), so instead of the whole x every rank receives,
        from each owner, only the overlap of [cmin, cmax] with the owner's x block -- straight into x_full, no packing.
        Otherwise (R-MAT: every rank reads every block) the whole x is assembled: by peer copies out of symmetric memory
        ("p2p") when that is available on CUDA, else by one NCCL all-gather."""
        world, blk = self.world, self.x_block
        self.recv_plan, self.send_plan, self.exchange = [], [], "allgather"
        if world == 1:
            return
        if exchange in ("auto", "halo"):
            if self.nnz > 0:
                cmin, cmax = int(self.col.min().item()), int(self.col.max().item()) + 1
            else:
                cmin, cmax = 0, 0
            need = torch.tensor([[cmin, cmax]], dtype=torch.int64, device=self.col.device)
            allneed = [torch.zeros_like(need) for _ in range(world)]
            dist.all_gather(allneed, need, group=self.group)
            ranges = [tuple(int(v) for v in t.flatten().tolist()) for t in allneed]      # (cmin, cmax) of every rank
            total = 0
            for g, (lo_need, hi_need) in enumerate(ranges):
                for h in range(world):
                    if h == g:
                        continue
                    lo, hi = max(lo_need, h * blk), min(hi_need, (h + 1) * blk)
                    if hi > lo:
                        total += hi - lo
                        if g == self.rank:
                            self.recv_plan.append((h, lo, hi))          # receive x[lo:hi] from its owner h
                        if h == self.rank:
                            self.send_plan.append((g, lo - h * blk, hi - h * blk))   # send my block[lo:hi] to g
            if exchange == "halo" or total * 2 < world * (world - 1) * blk:
                self.exchange = "halo"
                self.exchanged_elements = total
                return
        if exchange in ("auto", "p2p") and self.col.is_cuda and os.environ.get("B200SPMV_NO_P2P", "0") != "1":
            self.exchange = "p2p"

    def _init_p2p(self):
        """x shards in symmetric memory (two of them: step k writes shard k & 1), peer views, copy streams.  Any failure
        (no IPC support on the box, old driver) falls back to the NCCL all-gather -- decided collectively."""
        ok = 1
        try:
            import torch.distributed._symmetric_memory as symm
            grp = self.group if self.group is not None else dist.group.WORLD
            self.sym = [symm.empty(self.x_block, dtype=self.val.dtype, device=self.val.device) for _ in range(2)]
            self.hdl = [symm.rendezvous(t, group=grp) for t in self.sym]
            self.peer = [[h.get_buffer(r, (self.x_block,), self.val.dtype) for r in range(self.world)] for h in self.hdl]
            for t in self.sym:
                t.zero_()
            # flags of the device-side barrier (csrc/peer_sync.cu): one 8-byte slot per rank in every rank's buffer
            from . import lib as _lib
            self._L = _lib.shim()
            self.flags = symm.empty(self.world, dtype=torch.int64, device=self.val.device)
            self.flags.zero_()
            torch.cuda.synchronize()
            fh = symm.rendezvous(self.flags, group=grp)
            self._flag_views = [fh.get_buffer(r, (self.world,), torch.int64) for r in range(self.world)]
            self.flag_ptrs = torch.tensor([v.data_ptr() for v in self._flag_views], dtype=torch.int64, device=self.val.device)
            self.epoch = torch.zeros(1, dtype=torch.int64, device=self.val.device)
            torch.cuda.synchronize()
        except Exception as e:  # pragma: no cover (GPU boxes only)
            self.p2p_error = repr(e)
            ok = 0
        flag = torch.tensor([ok], dtype=torch.int32, device=self.val.device)
        dist.all_reduce(flag, op=dist.ReduceOp.MIN, group=self.group)
        if int(flag.item()) == 0:
            self.exchange = "allgather"
            self.side = torch.cuda.Stream()
            self.ev_in, self.ev_out = torch.cuda.Event(), torch.cuda.Event()
            return
        # Two copy streams, blocks issued IN ARRIVAL ORDER alternately on them: one copy-engine peer copy fills only part of
        # the NVLink ingress and splitting it over more streams does not help, so two copies in flight fill most of it
        # while the early blocks still land early (the panel pipeline below feeds on that).
        # B200SPMV_XCHG_SM_CTAS=n (> 0): pull the peer shards with an SM copy kernel of n CTAs (csrc/peer_sync.cu: LDG.128 from
        # peer memory over NVLink) instead of copy-engine copies
        self.sm_pull_ctas = int(os.environ.get("B200SPMV_XCHG_SM_CTAS", "0"))
        self.copy_streams = [torch.cuda.Stream() for _ in range(2)]
        self.own_stream = torch.cuda.Stream()
        self.ev_ready, self.ev_own = torch.cuda.Event(), torch.cuda.Event()
        self.ev_block = [torch.cuda.Event() for _ in range(self.world - 1)]

    def describe_exchange(self) -> str:
        if self.world == 1:
            return "none (single GPU)"
        if self.exchange == "halo":
            return f"halo exchange: {self.exchanged_elements * self.val.element_size()} B per step over all ranks (batch_isend_irecv)"
        how = {"p2p": "x shards in symmetric memory; one device-side barrier, then "
                      + (f"SM pull kernels ({self.sm_pull_ctas} CTAs, LDG.128 from peer memory)" if getattr(self, "sm_pull_ctas", 0) > 0 else "copy-engine peer copies")
                      + " over NVLink on side streams (double-buffered shards)",
               "allgather": "one NCCL all_gather_into_tensor on a side stream"}[self.exchange]
        if getattr(self, "_graphs", None):
            how += "; the whole step replayed as a CUDA graph"
        if self.panels:
            how += (f"; overlapped with the own-column panel of the local product ({self.own_nnz} of {self.nnz} local non-zeros), "
                    f"then {len(self.panel_groups) - 1} remote-column panel(s) in arrival order of their x blocks {self.panel_groups[1:]} "
                    "with beta = 1")
        return how

    # ------------------------------------------------------------------------------------------------ exchange
    def own_x_view(self) -> torch.Tensor:
        """This rank's block INSIDE the assembled x buffer.  A caller that keeps its x shard here (a CG driver its search
        direction) saves the staging copy of every product: the exchange then only has to bring in the other blocks."""
        blk = self.x_block
        return self.x_full[self.rank * blk:(self.rank + 1) * blk]

    def _stage_own(self, x_shard: torch.Tensor):
        own = self.own_x_view()
        if x_shard.data_ptr() != own.data_ptr():
            own.copy_(x_shard)

    def _halo_exchange(self, x_shard: torch.Tensor):
        blk = self.x_block
        self._stage_own(x_shard)
        ops = [dist.P2POp(dist.isend, x_shard[lo:hi], g, group=self.group) for g, lo, hi in self.send_plan]
        ops += [dist.P2POp(dist.irecv, self.x_full[lo:hi], h, group=self.group) for h, lo, hi in self.recv_plan]
        if ops:
            for w in dist.batch_isend_irecv(ops):
                w.wait()

    def _start_exchange(self, x_shard: torch.Tensor):
        """Kick off the assembly of x_full; returns the waits: one callable per panel (or a single one without panels) that
        makes the current stream wait until the x blocks of that panel are in place."""
        blk = self.x_block
        own = self.x_full[self.rank * blk:(self.rank + 1) * blk]
        if self.exchange == "p2p":
            i = self._step & 1
            self._step += 1
            main = torch.cuda.current_stream()
            if x_shard.data_ptr() != self.sym[i].data_ptr():
                self.sym[i].copy_(x_shard)                       # (a caller that produces its shard in shard_buffer() skips this)
            # every rank's shard i is written (and step k-1 is fully read): device-side barrier over NVLink peer memory,
            # epoch in device memory -> correct on every replay of a captured step; a missing rank traps after 30 s
            rc = self._L.b200peer_barrier(main.cuda_stream, self.flag_ptrs.data_ptr(), self.epoch.data_ptr(), self.rank, self.world,
                                          30.0)
            if rc != 0:
                raise RuntimeError(f"b200peer_barrier failed with code {rc}")
            self.ev_ready.record(main)
            self.own_stream.wait_event(self.ev_ready)
            with torch.cuda.stream(self.own_stream):              # my own block: a local copy next to the peer copies
                own.copy_(self.sym[i], non_blocking=True)
                self.ev_own.record(self.own_stream)
            for s in self.copy_streams:
                s.wait_event(self.ev_ready)
            for k, h in enumerate(self.pull_order):               # peer blocks in arrival order, alternating over two streams
                st = self.copy_streams[k & 1]
                with torch.cuda.stream(st):
                    if self.sm_pull_ctas > 0:
                        esz = self.x_full.element_size()
                        rc = self._L.b200peer_pull(st.cuda_stream, self.x_full.data_ptr() + h * blk * esz, self.peer[i][h].data_ptr(),
                                                   blk * esz, self.sm_pull_ctas)
                        if rc != 0:
                            raise RuntimeError(f"b200peer_pull failed with code {rc}")
                    else:
                        self.x_full[h * blk:(h + 1) * blk].copy_(self.peer[i][h], non_blocking=True)
                    self.ev_block[k].record(st)
            return self._p2p_waits(main)
        if self.exchange == "allgather" and hasattr(self, "side"):
            main = torch.cuda.current_stream()
            if x_shard.data_ptr() != own.data_ptr():
                own.copy_(x_shard)
            self.ev_in.record(main)
            self.side.wait_event(self.ev_in)
            with torch.cuda.stream(self.side):
                dist.all_gather_into_tensor(self.x_full, x_shard, group=self.group)
                self.ev_out.record(self.side)
            w = lambda: main.wait_event(self.ev_out)
            return [lambda: None] + [w] * (len(self.panel_groups) - 1) if self.panels else [w]
        # CPU (gloo tests) / no side stream: blocking exchange
        if x_shard.data_ptr() != own.data_ptr():
            own.copy_(x_shard)
        dist.all_gather_into_tensor(self.x_full, x_shard, group=self.group)
        return [lambda: None] * (len(self.panel_groups) if self.panels else 1)

    def _p2p_waits(self, main):
        """One wait per panel (own block, then each group of remote blocks), or a single wait for everything."""
        def wait_blocks(ks):
            def w():
                for k in ks:
                    main.wait_event(self.ev_block[k])
            return w
        if not self.panels:
            def wall():
                main.wait_event(self.ev_own)
                for e in self.ev_block:
                    main.wait_event(e)
            return [wall]
        waits, k = [lambda: main.wait_event(self.ev_own)], 0
        for g in self.panel_groups[1:]:
            waits.append(wait_blocks(list(range(k, k + len(g)))))
            k += len(g)
        return waits

    def shard_buffer(self):
        """p2p exchange: the symmetric-memory buffer the NEXT step publishes to the other ranks.  A caller that produces its
        x shard here (and passes this tensor as x_shard) saves the staging copy of the step."""
        if self.exchange != "p2p":
            raise RuntimeError("shard_buffer() exists for the p2p exchange only")
        return self.sym[self._step & 1]

    def new_x_shard(self, x=None):
        """This rank's equal block of a global vector x (zero-padded at the end of the last block)."""
        t = torch.zeros(self.x_block, dtype=self.val.dtype, device=self.val.device)
        if x is not None:
            lo = self.rank * self.x_block
            hi = min(lo + self.x_block, self.global_rows)
            if hi > lo:
                t[:hi - lo] = x[lo:hi]
        return t

    def new_y_shard(self, y=None):
        """This rank's row block of a global vector y."""
        t = torch.zeros(max(self.rows, 1), dtype=self.val.dtype, device=self.val.device)[:self.rows]
        if y is not None and self.rows:
            t.copy_(y[self.r0:self.r1])
        return t

    def gather_x(self, x_shard: torch.Tensor) -> torch.Tensor:
        """The path's single exchange step, complete on return (stream order): x_full holds everything this rank reads."""
        if self.world == 1:
            self._stage_own(x_shard)
        elif self.exchange == "halo":
            self._halo_exchange(x_shard)
        else:
            for w in self._start_exchange(x_shard):
                w()
        return self.x_full

    def spmv(self, x_shard: torch.Tensor, y_shard: torch.Tensor, alpha=1.0, beta=0.0) -> torch.Tensor:
        """y_shard = alpha * A[r0:r1, :] @ x + beta * y_shard   (x given as this rank's equal block)."""
        if not self.panels:
            self.gather_x(x_shard)
            if self.rows > 0:
                self.local_op(self.x_full, y_shard, alpha, beta)
            return y_shard
        waits = self._start_exchange(x_shard)
        for gi, (w, op) in enumerate(zip(waits, self.panel_ops)):  # own panel first; every later panel adds to y (beta = 1)
            w()
            op(self.x_full, y_shard, alpha, beta if gi == 0 else 1.0)
        return y_shard

    # ------------------------------------------------------------------------------------------------ SpMV + dot (CG)
    def can_fuse_dot(self) -> bool:
        """True when y = A x and y . x_shard can run as ONE kernel: the local matrix is whole (no column panels), lives on
        CUDA, has no row longer than csr_short_kernel takes, and the y rows coincide with this rank's x block (CG)."""
        if getattr(self, "_fuse_dot", None) is None:
            ok = (not self.panels) and self.val.is_cuda and self.rows > 0 and (self.rows == self.x_block or self.world == 1)
            if ok:
                try:
                    from . import lib as _lib
                    L = _lib.shim()
                    longest = int((self.off[1:] - self.off[:-1]).max().item())
                    ok = longest <= L.b200spmv_csr_short_max_row()
                    if ok:
                        self._dotL = L
                        self._dot_ws = torch.zeros(L.b200spmv_csr_short_dot_workspace_bytes(), dtype=torch.uint8, device=self.val.device)
                except Exception:
                    ok = False
            self._fuse_dot = bool(ok)
        return self._fuse_dot

    def spmv_dot(self, x_shard: torch.Tensor, y_shard: torch.Tensor, dot_out: torch.Tensor) -> torch.Tensor:
        """y_shard = A[r0:r1, :] @ x  and  dot_out[0] = y_shard . x_shard (this rank's part; fp64, device memory) in one pass
        over the local matrix: T = A*P together with T . P of a CG iteration (cg_example.c:220-227)."""
        assert self.can_fuse_dot()
        self.gather_x(x_shard)
        one = (C.c_double if self.val.dtype == torch.float64 else C.c_float)(1.0)
        zero = (C.c_double if self.val.dtype == torch.float64 else C.c_float)(0.0)
        rc = self._dotL.b200spmv_csr_short_mv_dot(torch.cuda.current_stream().cuda_stream, 1 if self.val.dtype == torch.float64 else 0,
                                                  self.rows, self.cols_padded, self.nnz, self.off.data_ptr(), self.col.data_ptr(),
                                                  self.val.data_ptr(), 0, C.byref(one), C.byref(zero), 0, self.x_full.data_ptr(),
                                                  y_shard.data_ptr(), x_shard.data_ptr(), dot_out.data_ptr(), self._dot_ws.data_ptr())
        if rc != 0:
            raise RuntimeError(f"b200spmv_csr_short_mv_dot failed with code {rc}")
        return y_shard

    def make_step(self, x_shard: torch.Tensor, y_shard: torch.Tensor, local_call=None, graph: bool | None = None,
                  in_place: bool = False):
        """A zero-argument callable for timing loops: one full step y = A x with fixed buffers and alpha = 1, beta = 0;
        uses the operators' prebuilt calls when they offer them (ctypes arguments built once).

        graph (default: on CUDA with panels): the step -- shard copies, device-side barrier, peer copies / all-gather on
        the side streams, both panel kernels -- is captured ONCE per shard-buffer parity into a CUDA graph and replayed:
        issued from Python the ~15 launches of a step cost more host time than the step
        takes on the GPUs.  If the capture is refused the eager step is returned and `self.graph_error` says why."""
        in_place = in_place and self.exchange == "p2p"
        if in_place:       # x does not change between the steps of this loop: it is published once, in both shard buffers
            for t in self.sym:
                t.copy_(x_shard)
        shard = (lambda: self.sym[self._step & 1]) if in_place else (lambda: x_shard)
        if not self.panels:
            call = local_call
            if call is None:
                op = self.local_op
                call = op.prebuilt(self.x_full, y_shard, 1.0, 0.0) if hasattr(op, "prebuilt") else (lambda: op(self.x_full, y_shard, 1.0, 0.0))
            if self.world == 1 or self.exchange == "halo":
                def step():
                    self.gather_x(x_shard)
                    call()
                return step

            def step():
                for w in self._start_exchange(shard()):
                    w()
                call()
            return self._maybe_graph(step, x_shard, graph)
        mk = lambda op, beta: (op.prebuilt(self.x_full, y_shard, 1.0, beta) if hasattr(op, "prebuilt")
                               else (lambda op=op: op(self.x_full, y_shard, 1.0, beta)))
        calls = [mk(op, 0.0 if gi == 0 else 1.0) for gi, op in enumerate(self.panel_ops)]
        self.panel_calls = calls

        def step():
            for w, call in zip(self._start_exchange(shard()), calls):
                w()
                call()
        return self._maybe_graph(step, x_shard, graph)

    def _maybe_graph(self, step, x_shard, graph):
        if graph is None:   # (NCCL inside a captured step is slower than eager -- graphs only for p2p)
            graph = x_shard.is_cuda and self.exchange == "p2p" and os.environ.get("B200SPMV_STEP_GRAPH", "1") != "0"
        if not graph:
            return step
        try:
            return self._graphed_step(step)
        except Exception as e:   # pragma: no cover (GPU boxes only)
            self.graph_error = repr(e)
            torch.cuda.synchronize()
            return step

    def _graphed_step(self, step):
        """Two graphs, one per parity of the double-buffered x shard (the p2p exchange alternates buffers so that one
        barrier per step suffices); replayed alternately in the order the eager steps would run."""
        main = torch.cuda.current_stream()
        cap = torch.cuda.Stream()
        ops = [op for op in (self.panel_ops if self.panels else (self.local_op,)) if hasattr(op, "handle")]
        for _ in range(2):                      # warm-up: both parities, eagerly, on the stream the graphs are captured on
            step()
        torch.cuda.synchronize()
        graphs = []
        nparity = 2 if self.exchange == "p2p" else 1
        cap.wait_stream(main)
        try:
            with torch.cuda.stream(cap):
                for op in ops:
                    op.api.cusparseSetStream(op.handle, cap.cuda_stream)
                for _ in range(2):
                    step()
                cap.synchronize()
                for i in range(nparity):
                    g = torch.cuda.CUDAGraph()
                    with torch.cuda.graph(g, stream=cap):
                        step()
                    graphs.append(g)
        finally:
            for op in ops:                      # the operators go back to the caller's stream whatever happened
                op.api.cusparseSetStream(op.handle, main.cuda_stream)
        main.wait_stream(cap)
        torch.cuda.synchronize()
        if self.world > 1:
            dist.barrier(group=self.group)
        self._graphs, self._gi = graphs, 0
        self.graph_error = None

        def replay():
            self._graphs[self._gi].replay()
            self._gi = (self._gi + 1) % len(self._graphs)
        return replay

    def close(self):
        if getattr(self, "_graphs", None):
            torch.cuda.synchronize()
            self._graphs = None
        for op in (self.panel_ops if self.panels else [self.local_op]):
            if op is not None and hasattr(op, "close"):
                op.close()
