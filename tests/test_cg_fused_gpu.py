"""GPU: the fused CG BLAS-1 kernels of cg_fused.cu (b200cg_dot, _update_r, _update_xr, _update_xp, _update_p), BIT FOR BIT.

On the exact fixtures of oracle/exact.py (nonzero integer vectors, alpha = -1/4 and beta = 1/2 from the device scalars) every
updated element and every partial sum of a reduction is exact, so each kernel must return the int64 reference whatever its
summation order.  The sizes sit on the kernels' borders (oracle.exact.cg_sizes: the odd scalar tail in the first and in a
later grid-stride pass, one and two CTAs, the grid cap, one full pass F, several passes); the coverage of those classes is
checked on the CPU in test_exact_fixtures.py.

Every call goes through the C ABI on the torch current stream.  Around each call: the scalar outputs are NaN beforehand (a
missing write shows), every vector is a 16-byte aligned view with NaN guard elements on both sides (a write outside [0, n)
shows), and the arrival counter of the workspace must be back at 0 afterwards.  Then: one workspace shared by launches of
different grids, determinism and the summation error bound on inexact data (also under CUDA-graph replay), and the host-side
argument checks."""
import ctypes as C
import math

import numpy as np
import pytest
import torch

from oracle import exact as E

pytestmark = pytest.mark.gpu

LEAD, TRAIL = 2, 3                                   # guard elements; LEAD = 2 keeps the view 16-byte aligned
GUARD = np.uint64(0x7FF8DEAD0BAD0001)                # a quiet NaN with a payload no kernel produces
SLOT = {"delta": 0, "denom": 1, "delta_new": 2, "out": 3}


@pytest.fixture(scope="module")
def L():
    from cudalibrarysamples_b200 import lib as _lib
    lib = _lib.shim()
    return lib


@pytest.fixture(scope="module")
def P(L):
    return E.cg_params(L)


@pytest.fixture
def ws(L):
    return torch.zeros(int(L.b200cg_workspace_bytes()), dtype=torch.uint8, device="cuda")


def counter(ws, P):
    """the arrival counter: uint32 at byte max_ctas * 8 of the workspace"""
    off = P["max_ctas"] * 8
    return int(ws[off:off + 4].cpu().numpy().view(np.uint32)[0])


def guarded(values):
    """(allocation, view): the float64 values LEAD elements into a NaN-guarded device allocation"""
    n = len(values)
    host = np.empty(LEAD + n + TRAIL, np.float64)
    host.view(np.uint64)[:] = GUARD
    host[LEAD:LEAD + n] = values
    buf = torch.from_numpy(host).cuda()
    return buf, buf[LEAD:LEAD + n]


def guards_intact(buf, n):
    bits = buf.cpu().numpy().view(np.uint64)
    return bool(np.all(bits[:LEAD] == GUARD) and np.all(bits[LEAD + n:] == GUARD))


def scalars(delta_new_is_input=True):
    s = torch.tensor([E.CG_SCALARS["delta"], E.CG_SCALARS["denom"], E.CG_SCALARS["delta_new"], float("nan")],
                     dtype=torch.float64, device="cuda")
    if not delta_new_is_input:
        s[SLOT["delta_new"]] = float("nan")
    return s


def addr(t):
    return t.data_ptr()


def call(L, name, n, vec_ptrs, scal, ws, override=None):
    """b200cg_<name>(stream, n, vectors..., device scalars..., [workspace]) on the current stream; override: {argument
    name: raw address or None} replaces single pointers"""
    k = E.CG_KERNELS[name]
    ptrs = dict(zip(k.vectors, vec_ptrs))
    ptrs.update({s: scal.data_ptr() + 8 * SLOT[s] for s in k.scalars})
    if k.workspace:
        ptrs["ws"] = ws.data_ptr()
    ptrs.update(override or {})
    order = k.vectors + k.scalars + (["ws"] if k.workspace else [])
    stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    return getattr(L, "b200cg_" + name)(stream, C.c_int64(n), *[C.c_void_p(ptrs[a]) for a in order])


def run_exact(L, P, ws, name, n, v):
    """one call on guarded copies of the int64 vectors v: {written vector / reduced scalar: float64 result}; asserts the
    return code, the guard elements, the untouched inputs and the counter"""
    k = E.CG_KERNELS[name]
    bufs = {a: guarded(v[a].astype(np.float64)) for a in k.vectors}
    scal = scalars(delta_new_is_input=k.reduces != "delta_new")
    assert call(L, name, n, [addr(bufs[a][1]) for a in k.vectors], scal, ws) == 0
    torch.cuda.synchronize()
    out = {}
    for a, (buf, view) in bufs.items():
        assert guards_intact(buf, n), f"{name} n={n}: a guard element of {a} was overwritten"
        got = view.cpu().numpy()
        if a in k.writes:
            out[a] = got
        else:
            assert np.array_equal(got, v[a].astype(np.float64)), f"{name} n={n}: input {a} changed"
    if k.reduces:
        out[k.reduces] = float(scal[SLOT[k.reduces]].item())
    if k.workspace:
        assert counter(ws, P) == 0, f"{name} n={n}: arrival counter left at {counter(ws, P)}"
    return out


def assert_equal(got, want, what):
    for key, w in want.items():
        g = got[key]
        if isinstance(w, float):
            assert g == w, f"{what}: {key} = {g!r}, want {w!r}"
        elif not np.array_equal(g, w):
            bad = np.flatnonzero(g != w)
            raise AssertionError(f"{what}: {key}: {bad.size} of {w.size} elements differ, first at {bad[:5].tolist()}: "
                                 f"got {g[bad[:5]].tolist()} want {w[bad[:5]].tolist()}")


# ------------------------------------------------------------------------------------------ exact results at every edge size
@pytest.mark.parametrize("kind", E.CG_KINDS)
@pytest.mark.parametrize("name", list(E.CG_KERNELS))
def test_exact_at_every_edge_size(L, P, ws, name, kind):
    for n in E.cg_sizes(P):
        v = E.cg_vectors(kind, n, E.CG_KERNELS[name].vectors, seed=n)
        assert_equal(run_exact(L, P, ws, name, n, v), E.cg_reference(name, v), f"{name} {kind} n={n}")


def test_one_workspace_shared_by_grids_of_every_size(L, P, ws):
    """The partial-sum slots and the counter are reused by launches whose grids grow and shrink; nothing of a previous
    launch may leak into the next result."""
    P2, F = 2 * P["block"], E.cg_full_pass(P)
    seq = [("dot", 3 * F + P2 + 1), ("update_r", 5), ("dot", F + 1), ("update_xr", P2 + 1), ("dot", 0), ("update_r", 2 * F + 3),
           ("dot", 33), ("update_xr", F), ("dot", 1), ("update_p", 2 * P2 + 1), ("dot", 2 * F)]
    for i, (name, n) in enumerate(seq):
        for kind in E.CG_KINDS:
            v = E.cg_vectors(kind, n, E.CG_KERNELS[name].vectors, seed=100 + i)
            assert_equal(run_exact(L, P, ws, name, n, v), E.cg_reference(name, v), f"step {i}: {name} {kind} n={n}")


# ------------------------------------------------------------------------------------------ inexact data: bound and determinism
def mantissa26(rng, n):
    """random doubles with 26-bit significands: every product of two is exact in fp64"""
    m = rng.integers(1 << 25, 1 << 26, n, dtype=np.int64) * rng.choice(np.array([-1, 1], np.int64), n)
    return np.ldexp(m.astype(np.float64), rng.integers(-40, -20, n))


def test_dot_is_accurate_and_deterministic_with_and_without_graph_replay(L, P, ws):
    P2, F = 2 * P["block"], E.cg_full_pass(P)
    u = 2.0 ** -53
    for n in (33, 5 * P2 + 1, F - 1, F + 1, 3 * F + P2 + 1):
        rng = np.random.default_rng(n)
        a, b = mantissa26(rng, n), mantissa26(rng, n)
        prod = a * b                                                       # exact
        ref, mag = math.fsum(prod), math.fsum(np.abs(prod))
        w = E.cg_walk(n, P)
        K = 2 * w["passes"] + 5 + 8 + w["grid"]                            # per-thread adds, warp shuffles, warps, CTAs
        gamma = K * u / (1 - K * u)
        da, db = torch.from_numpy(a).cuda(), torch.from_numpy(b).cuda()
        scal = scalars()
        bits = []
        for _ in range(3):
            scal[SLOT["out"]] = float("nan")
            assert call(L, "dot", n, [addr(da), addr(db)], scal, ws) == 0
            bits.append(scal[SLOT["out"]:SLOT["out"] + 1].view(torch.int64).item())
            assert counter(ws, P) == 0
        got = float(scal[SLOT["out"]].item())
        assert abs(got - ref) <= gamma * mag, (n, got, ref, gamma * mag)
        assert bits == [bits[0]] * 3, f"n={n}: three calls gave {bits}"
        # the same call captured in a CUDA graph and replayed twice gives the same bits
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            assert call(L, "dot", n, [addr(da), addr(db)], scal, ws) == 0
        for _ in range(2):
            scal[SLOT["out"]] = float("nan")
            g.replay()
            torch.cuda.synchronize()
            assert scal[SLOT["out"]:SLOT["out"] + 1].view(torch.int64).item() == bits[0], f"n={n}: graph replay differs"
            assert counter(ws, P) == 0
        del g


# ------------------------------------------------------------------------------------------ argument checks
@pytest.mark.parametrize("name", list(E.CG_KERNELS))
def test_invalid_arguments_launch_nothing(L, P, ws, name):
    """n < 0, a required pointer NULL while n > 0, a vector one element off its 16-byte alignment: -1, and no kernel ran
    (outputs still NaN, vectors unchanged, counter 0).  n = 0 with NULL vectors is valid and reduces to exactly 0."""
    k = E.CG_KERNELS[name]
    n = 2 * P["block"] + 7
    v = E.cg_vectors("f64", n, k.vectors, seed=5)
    bufs = {a: guarded(v[a].astype(np.float64)) for a in k.vectors}
    ptrs = [addr(bufs[a][1]) for a in k.vectors]
    cases = [("n = -1", -1, {})]
    cases += [(f"{a} = NULL", n, {a: None}) for a in k.vectors + k.scalars + (["ws"] if k.workspace else [])]
    cases += [(f"{a} + 8 bytes", n, {a: addr(bufs[a][1]) + 8}) for a in k.vectors]
    for what, nn, override in cases:
        scal = scalars(delta_new_is_input=k.reduces != "delta_new")
        assert call(L, name, nn, ptrs, scal, ws, override) == -1, f"{name}: {what} accepted"
        torch.cuda.synchronize()
        if k.reduces:
            assert math.isnan(scal[SLOT[k.reduces]].item()), f"{name}: {what} wrote {k.reduces}"
        for a, (buf, view) in bufs.items():
            assert np.array_equal(view.cpu().numpy(), v[a].astype(np.float64)) and guards_intact(buf, n), f"{name}: {what} wrote {a}"
        assert counter(ws, P) == 0
    # n = 0: the vectors may be NULL; a reduction still writes its (empty) sum
    scal = scalars(delta_new_is_input=k.reduces != "delta_new")
    assert call(L, name, 0, ptrs, scal, ws, {a: None for a in k.vectors}) == 0
    torch.cuda.synchronize()
    if k.reduces:
        got = scal[SLOT[k.reduces]:SLOT[k.reduces] + 1]
        assert got.view(torch.int64).item() == 0, f"{name}: n = 0 gave {got.item()!r}, want +0.0"
        assert counter(ws, P) == 0
