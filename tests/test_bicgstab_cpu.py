"""CPU: the BiCGStab restatement, the torch-op driver under gloo, the C ABI's layout and argument checks, the exact fixtures'
size coverage, and the unchanged SASS of the CG kernels whose reduction helpers BiCGStab now shares."""
import ctypes as C
import hashlib
import json
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import scipy.sparse as sp
import scipy.sparse.linalg as spla
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from oracle import bicgstab_ref as BR
from oracle import exact as E
from oracle import oracle as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def sample_system(grid):
    """the sample's advection-diffusion operator (bicgstab_example.c's matrix: mass 0.3, ux 0.3, uy 0.2), b = 0.75 A 1"""
    off, col, val = O.gen_stencil5(grid, 0.3, 0.3, 0.2)
    n = grid * grid
    A = sp.csr_matrix((val, col, off), shape=(n, n))
    return A, 0.75 * (A @ np.ones(n))


def dominant_nonsymmetric(n, seed):
    rng = np.random.default_rng(seed)
    A = sp.random(n, n, density=min(1.0, 6.0 / n), random_state=seed, format="csr") * 2.0 - sp.random(
        n, n, density=min(1.0, 4.0 / n), random_state=seed + 1, format="csr")
    A = A + sp.diags(np.abs(A).sum(axis=1).A1 + 1.0 + rng.random(n))
    return A.tocsr(), rng.standard_normal(n)


# ------------------------------------------------------------------------------------------ the restatement
SYSTEMS = {"sample_20": lambda: sample_system(20), "sample_33": lambda: sample_system(33),
           "dominant_200": lambda: dominant_nonsymmetric(200, 3), "dominant_517": lambda: dominant_nonsymmetric(517, 8)}


@pytest.mark.parametrize("name", list(SYSTEMS))
def test_restatement_is_the_sample_loop_bit_for_bit(name):
    A, b = SYSTEMS[name]()
    for tol in (1e-6, 1e-10, 1e-14):
        want = BR.sample_loop(A, b, 400, tol)
        got = BR.fused(lambda v: A @ v, b, 400, tol)
        assert want["exit"] is not None, (name, tol, "the sample loop did not converge")
        assert got["status"] == {"s": BR.CONVERGED_S, "r": BR.CONVERGED_R}[want["exit"]]
        assert got["iterations"] == want["iterations"]
        assert got["history"] == want["history"]
        assert np.array_equal(got["x"], want["x"]), (name, tol)


@pytest.mark.parametrize("name", list(SYSTEMS))
def test_restatement_solves_like_spsolve(name):
    A, b = SYSTEMS[name]()
    got = BR.fused(lambda v: A @ v, b, 1000, 1e-12)
    assert got["status"] in (BR.CONVERGED_S, BR.CONVERGED_R)
    ref = spla.spsolve(A.tocsc(), b)
    assert np.linalg.norm(got["x"] - ref) <= 1e-9 * np.linalg.norm(ref)
    assert np.linalg.norm(b - A @ got["x"]) <= 10 * 1e-12 * np.linalg.norm(b)


def test_restatement_status_protocol():
    # skew-symmetric tridiagonal, integer b: r0 . A r0 = 0 exactly, the denominator breaks down in iteration 1, x stays 0
    n = 64
    A = sp.diags([np.ones(n - 1), -np.ones(n - 1)], [1, -1], format="csr")
    b = E.nonzero_ints(np.random.default_rng(1), n, 1, 5).astype(np.float64)
    got = BR.fused(lambda v: A @ v, b, 50, 1e-10)
    assert got["status"] == BR.BREAKDOWN_DENOM and got["iterations"] == 0 and not np.any(got["x"])
    # tol = None: exactly max_iters iterations
    A, b = sample_system(12)
    got = BR.fused(lambda v: A @ v, b, 7, None)
    assert got["status"] == BR.RUNNING and got["iterations"] == 7 and len(got["history"]) == 8
    # b = 0: converged before the first iteration
    got = BR.fused(lambda v: A @ v, np.zeros_like(b), 7, 1e-8)
    assert got["status"] == BR.CONVERGED_R and got["iterations"] == 0
    # the identity: s = 0 after one step, converged at s
    I = sp.identity(30, format="csr")
    got = BR.fused(lambda v: I @ v, np.arange(1.0, 31.0), 10, 1e-12)
    assert got["status"] == BR.CONVERGED_S and got["iterations"] == 1 and np.array_equal(got["x"], np.arange(1.0, 31.0))


def test_status_codes_and_slots_match_the_header():
    from cudalibrarysamples_b200 import bicgstab as B
    text = open(os.path.join(ROOT, "include", "b200spmv.h")).read()
    defs = {m.group(1): int(m.group(2)) for m in re.finditer(r"#define B200BICGSTAB_(\w+)\s+(\d+)", text)}
    for code, name in BR.STATUS_NAMES.items():
        assert defs[name.upper()] == code and B.STATUS_NAMES[code] == name
    for slot, idx in BR.SLOTS.items():
        assert defs[slot] == idx and getattr(B, slot) == idx


# ------------------------------------------------------------------------------------------ the torch-op driver under gloo
def _free_port():
    import socket
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _collect(q, procs, timeout=240):
    """the result rank 0 put on the queue, or a test failure (not a hang) when a worker died or the time is up"""
    import time
    t0 = time.time()
    while q.empty():
        if any(p.exitcode not in (None, 0) for p in procs) or time.time() - t0 > timeout:
            for p in procs:
                p.kill()
            pytest.fail("a worker failed or timed out: " + str([p.exitcode for p in procs]))
        time.sleep(0.05)
    return q.get()


def _oracle_op(rows, cols, arrays):
    off, col, val = (arrays[k].numpy() for k in ("off", "col", "val"))

    def op(x, y, alpha, beta):
        y.copy_(torch.from_numpy(O.spmv_csr(off, col, val, x.numpy(), y.numpy(), alpha, beta)))
        return y
    return op


def _worker(rank, world, port, grid, q):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from cudalibrarysamples_b200.bicgstab import make_bicgstab_solver
        from cudalibrarysamples_b200.sharded import ShardedCsr
        off, col, val = (torch.from_numpy(a) for a in O.gen_stencil5(grid, 0.3, 0.3, 0.2))
        n = grid * grid
        sh = ShardedCsr(off, col, val, rank, world, _oracle_op, balance="rows")
        b = sh.new_y_shard()
        sh.spmv(sh.new_x_shard(torch.ones(n, dtype=torch.float64)), b, alpha=0.75, beta=0.0)
        res = make_bicgstab_solver(sh, b).run(500, 1e-10)
        out = [None] * world
        dist.all_gather_object(out, dict(rank=rank, x=res.x.numpy(), status=res.status, iterations=res.iterations,
                                         history=res.history))
        if rank == 0:
            q.put(out)
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("world", [1, 2, 4])
def test_sharded_bicgstab_matches_the_restatement(world):
    grid = 24
    ctx = mp.get_context("spawn")
    q = ctx.SimpleQueue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, world, port, grid, q)) for r in range(world)]
    for p in procs:
        p.start()
    out = _collect(q, procs)
    for p in procs:
        p.join(60)
        assert p.exitcode == 0
    out.sort(key=lambda d: d["rank"])
    A, b = sample_system(grid)
    want = BR.fused(lambda v: A @ v, b, 500, 1e-10)
    assert want["status"] in (BR.CONVERGED_S, BR.CONVERGED_R)
    for d in out:
        assert d["status"] == BR.STATUS_NAMES[want["status"]] and d["iterations"] == want["iterations"]
    x = np.concatenate([d["x"] for d in out])
    assert np.linalg.norm(x - want["x"]) <= 1e-9 * np.linalg.norm(want["x"])
    np.testing.assert_allclose(out[0]["history"], want["history"], rtol=1e-6)


# ------------------------------------------------------------------------------------------ C ABI without a device
@pytest.fixture(scope="module")
def L():
    from cudalibrarysamples_b200 import lib as _lib
    return _lib.shim()


def test_layout_and_workspace(L):
    P = E.cg_params(L)
    assert L.b200bicgstab_workspace_bytes() == (2 * P["max_ctas"] + 2) * 8 >= L.b200cg_workspace_bytes()
    sb, ib, hb = C.c_int32(), C.c_int32(), C.c_int32()
    assert L.b200bicgstab_state_layout(0, C.byref(sb), C.byref(ib), C.byref(hb)) == hb.value == 96
    assert (sb.value, ib.value) == (80, 84)
    assert L.b200bicgstab_state_layout(201, None, None, None) == 96 + 201 * 8
    assert L.b200bicgstab_state_layout(-1, None, None, None) == 0 and L.b200bicgstab_state_layout(1 << 31, None, None, None) == 0


def test_invalid_arguments_are_rejected_before_any_launch(L):
    """every rejection happens on the host: these calls touch no device (this machine may have none)"""
    a16, a8 = 1 << 20, (1 << 20) + 8                   # fake addresses, never dereferenced
    s = 0
    assert L.b200bicgstab_init(s, -1, a16, a16, a16, a16, 1, 1e-8) == -1
    assert L.b200bicgstab_init(s, 4, a16, a16, a16, None, 1, 1e-8) == -1
    assert L.b200bicgstab_init(s, 4, a16, a16, a8, a16, 1, 1e-8) == -1
    assert L.b200bicgstab_init(s, 4, a16, a16, a16, a16, -1, 1e-8) == -1
    assert L.b200bicgstab_init(s, 4, a16, a16, a16, a16, 1, float("nan")) == -1
    assert L.b200bicgstab_update_s(s, 4, a16, a16, a16, a16, None) == -1
    assert L.b200bicgstab_update_s(s, 4, a16, None, a16, a16, a16) == -1
    assert L.b200bicgstab_dot2(s, -3, a16, a16, a16, a16) == -1
    assert L.b200bicgstab_dot2(s, 4, a16, a16, a8, a16) == -1
    assert L.b200bicgstab_update_xr(s, 4, a16, a16, a16, a16, a16, None, a16, a16) == -1
    assert L.b200bicgstab_update_xr(s, 4, a16, a16, a16, a8, a16, a16, a16, a16) == -1
    assert L.b200bicgstab_update_p(s, 4, a16, a16, a16, None) == -1
    assert L.b200bicgstab_update_p(s, 4, a16, a8, a16, a16) == -1


# ------------------------------------------------------------------------------------------ exact fixtures
def test_exact_fixtures_cover_every_size_class_and_stay_exact(L):
    P = E.cg_params(L)
    hit = set()
    for n in E.cg_sizes(P):
        hit |= E.cg_coverage(n, P)
        for name in BR.KERNELS:
            for kind in E.CG_KINDS:
                BR.kernel_reference(name, BR.kernel_vectors(kind, n, name, seed=n), BR.kernel_scalars(name))  # asserts exactness
    assert hit == set(E.CG_CLASSES), set(E.CG_CLASSES) - hit


# ------------------------------------------------------------------------------------------ CG's kernels did not change
def _sass_fingerprints(src, flags, workdir):
    cubin = os.path.join(workdir, "k.cubin")
    subprocess.check_call([shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc", *flags.split(), "-o", cubin, src])
    cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    out = subprocess.check_output([cuobjdump, "-sass", cubin], text=True)
    funcs, cur = {}, None
    for line in out.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            cur = m.group(1)
            funcs[cur] = []
        elif cur and line.strip():
            funcs[cur].append(line.strip())
    return {k: hashlib.sha256("\n".join(v).encode()).hexdigest() for k, v in funcs.items()}


def test_cg_kernels_compile_to_the_same_sass(tmp_path):
    golden = json.load(open(os.path.join(ROOT, "tests", "golden", "cg_fused_sass.json")))
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("no nvcc")
    if golden["nvcc"] not in subprocess.check_output([nvcc, "--version"], text=True):
        pytest.skip("the fingerprints were taken with " + golden["nvcc"])
    got = _sass_fingerprints(os.path.join(ROOT, "cudalibrarysamples_b200", "csrc", "cg_fused.cu"), golden["flags"], str(tmp_path))
    assert got == golden["kernels"]
