"""GPU: the fused BiCGStab kernels of bicgstab_fused.cu through the C ABI, bit for bit on the exact fixtures of
oracle/bicgstab_ref.py at every size of oracle.exact.cg_sizes (NaN guards on both sides of every vector, inputs unchanged,
arrival counter back at 0); every status transition from hand-set scalars, and the frozen state in which every kernel is a
no-op; and FusedBicgstabSolver on the sample's system, against the numpy restatement, on both launch paths."""
import ctypes as C
import math

import numpy as np
import pytest
import scipy.sparse as sp
import scipy.sparse.linalg as spla
import torch

from oracle import bicgstab_ref as BR
from oracle import exact as E
from oracle import oracle as O

pytestmark = pytest.mark.gpu

LEAD, TRAIL = 2, 3
GUARD = np.uint64(0x7FF8DEAD0BAD0001)


@pytest.fixture(scope="module")
def L():
    from cudalibrarysamples_b200 import lib as _lib
    return _lib.shim()


@pytest.fixture(scope="module")
def P(L):
    return E.cg_params(L)


@pytest.fixture
def ws(L):
    return torch.zeros(int(L.b200bicgstab_workspace_bytes()), dtype=torch.uint8, device="cuda")


def counter(ws, P):
    off = P["max_ctas"] * 8
    return int(ws[off:off + 4].cpu().numpy().view(np.uint32)[0])


def guarded(values):
    n = len(values)
    host = np.empty(LEAD + n + TRAIL, np.float64)
    host.view(np.uint64)[:] = GUARD
    host[LEAD:LEAD + n] = values
    buf = torch.from_numpy(host).cuda()
    return buf, buf[LEAD:LEAD + n]


def guards_intact(buf, n):
    bits = buf.cpu().numpy().view(np.uint64)
    return bool(np.all(bits[:LEAD] == GUARD) and np.all(bits[LEAD + n:] == GUARD))


def new_state(L, scal, status=BR.RUNNING, cap=4):
    st = torch.zeros(L.b200bicgstab_state_layout(cap, None, None, None) // 8, dtype=torch.float64, device="cuda")
    for k, v in scal.items():
        st[BR.SLOTS[k]] = v
    st.view(torch.int32)[20] = status
    st.view(torch.int32)[22] = cap
    st[12:] = float("nan")
    return st


def status_of(st):
    return int(st.view(torch.int32)[20].item())


def iters_of(st):
    return int(st.view(torch.int32)[21].item())


def call(L, name, n, ptrs, st, ws, tol=-1.0):
    s = torch.cuda.current_stream().cuda_stream
    f = getattr(L, "b200bicgstab_" + name)
    if name == "init":
        return f(s, n, *ptrs, st.data_ptr(), (st.numel() * 8 - 96) // 8, tol)
    if name == "update_p":
        return f(s, n, *ptrs, st.data_ptr())
    return f(s, n, *ptrs, st.data_ptr(), ws.data_ptr())


# ------------------------------------------------------------------------------------------ exact, at every edge size
@pytest.mark.parametrize("kind", E.CG_KINDS)
@pytest.mark.parametrize("name", list(BR.KERNELS))
def test_exact_at_every_edge_size(L, P, ws, name, kind):
    names, writes, reduces = BR.KERNELS[name]
    for n in E.cg_sizes(P):
        v = BR.kernel_vectors(kind, n, name, seed=n)
        want = BR.kernel_reference(name, v)
        bufs = {a: guarded(v[a].astype(np.float64)) for a in names}
        scal = dict(BR.kernel_scalars(name))
        if name == "init":
            scal = dict(RHO_NEW=16.0)
        st = new_state(L, scal)
        for k in reduces:
            st[BR.SLOTS[k]] = float("nan")
        assert call(L, name, n, [bufs[a][1].data_ptr() for a in names], st, ws, tol=0.5) == 0
        torch.cuda.synchronize()
        for a, (buf, view) in bufs.items():
            assert guards_intact(buf, n), f"{name} n={n}: a guard of {a} was overwritten"
            got = view.cpu().numpy()
            if a in writes:
                assert np.array_equal(got, want[a]), f"{name} {kind} n={n}: {a} differs"
            else:
                assert np.array_equal(got, v[a].astype(np.float64)), f"{name} n={n}: input {a} changed"
        for k in reduces:
            assert float(st[BR.SLOTS[k]].item()) == want[k], f"{name} {kind} n={n}: {k} = {st[BR.SLOTS[k]].item()} want {want[k]}"
        assert status_of(st) == BR.RUNNING
        assert counter(ws, P) == 0, f"{name} n={n}: arrival counter left at {counter(ws, P)}"
        if name == "update_s":
            assert st[BR.SLOTS["ALPHA"]].item() == -0.25 and st[BR.SLOTS["RHO"]].item() == scal["RHO_NEW"]
        if name == "update_xr":
            assert st[BR.SLOTS["OMEGA"]].item() == 0.5
        if name == "update_p":
            assert iters_of(st) == 1
        if name == "init":
            h = st[12:].cpu().numpy()
            assert st[BR.SLOTS["RHO"]].item() == 16.0 and st[BR.SLOTS["R2"]].item() == 16.0 and iters_of(st) == 0
            assert st[BR.SLOTS["THRESHOLD"]].item() == 2.0 and h[0] == 4.0


# ------------------------------------------------------------------------------------------ status transitions
N = 3001


def vectors(seed):
    rng = np.random.default_rng(seed)
    return {k: torch.from_numpy(E.nonzero_ints(rng, N, 1, 5).astype(np.float64)).cuda() for k in ("x", "r", "p", "s", "t", "r0", "v")}


def snapshot(vs, st):
    return {k: t.clone() for k, t in vs.items()}, st.clone()


def unchanged(before, vs, st):
    vb, sb = before
    return all(torch.equal(vb[k].view(torch.int64), vs[k].view(torch.int64)) for k in vs) and torch.equal(
        sb.view(torch.int64), st.view(torch.int64))


def run_kernel(L, name, vs, st, ws):
    ptrs = {"update_s": ["r", "v", "s"], "dot2": ["t", "s"], "update_xr": ["x", "r", "p", "s", "t", "r0"], "update_p": ["p", "r", "v"]}[name]
    assert call(L, name, N, [vs[a].data_ptr() for a in ptrs], st, ws) == 0
    torch.cuda.synchronize()


@pytest.mark.parametrize("case", ["denom", "nonfinite_alpha", "tt", "omega", "nonfinite_s2", "rho", "nonfinite_r2"])
def test_breakdowns_update_nothing(L, P, ws, case):
    kernel, scal = {
        "denom": ("update_s", dict(BR.SCALARS, DENOM=0.0)),
        "nonfinite_alpha": ("update_s", dict(BR.SCALARS, DENOM=1e-320, RHO_NEW=1e300)),
        "tt": ("update_xr", dict(BR.SCALARS, TT=0.0, TS=0.0)),
        "omega": ("update_xr", dict(BR.SCALARS, TS=0.0)),
        "nonfinite_s2": ("update_xr", dict(BR.SCALARS, S2=float("inf"))),
        "rho": ("update_p", dict(BR.SCALARS_P, RHO_NEW=0.0)),
        "nonfinite_r2": ("update_p", dict(BR.SCALARS_P, R2=float("nan"))),
    }[case]
    want = {"denom": BR.BREAKDOWN_DENOM, "tt": BR.BREAKDOWN_TT, "omega": BR.BREAKDOWN_OMEGA, "rho": BR.BREAKDOWN_RHO}.get(
        case, BR.BREAKDOWN_NONFINITE)
    vs = vectors(1)
    st = new_state(L, scal)
    before = snapshot(vs, st)
    run_kernel(L, kernel, vs, st, ws)
    assert status_of(st) == want
    assert all(torch.equal(before[0][k], vs[k]) for k in vs), f"{case}: a vector changed"
    # only the status word (and, for update_p, the counter and history entry of the finished iteration) changed
    stb = before[1].clone()
    stb.view(torch.int32)[20] = want
    if kernel == "update_p":
        stb.view(torch.int32)[21] = 1
        stb[13] = st[13]
    assert torch.equal(stb.view(torch.int64), st.view(torch.int64)), case
    assert counter(ws, P) == 0


def test_converged_at_s_and_at_r(L, P, ws):
    # at s: x += alpha p, r = s, r0 . r and r . r reduced, counter 1, history[1] = sqrt(s2)
    vs = vectors(2)
    st = new_state(L, dict(BR.SCALARS, S2=4.0, THRESHOLD=2.5))
    x0, p, s, r0 = (vs[k].cpu().numpy().copy() for k in ("x", "p", "s", "r0"))
    run_kernel(L, "update_xr", vs, st, ws)
    assert status_of(st) == BR.CONVERGED_S and iters_of(st) == 1 and st[13].item() == 2.0
    assert np.array_equal(vs["x"].cpu().numpy(), x0 - p / 4) and np.array_equal(vs["r"].cpu().numpy(), s)
    assert st[BR.SLOTS["RHO_NEW"]].item() == float(np.dot(r0.astype(np.int64), s.astype(np.int64)))
    assert st[BR.SLOTS["R2"]].item() == float(np.dot(s.astype(np.int64), s.astype(np.int64)))
    assert counter(ws, P) == 0
    # at r: p untouched, counter 1, history[1] = sqrt(r2)
    vs = vectors(3)
    st = new_state(L, dict(BR.SCALARS_P, R2=9.0, THRESHOLD=3.5))
    p0 = vs["p"].clone()
    run_kernel(L, "update_p", vs, st, ws)
    assert status_of(st) == BR.CONVERGED_R and iters_of(st) == 1 and st[13].item() == 3.0 and torch.equal(vs["p"], p0)


@pytest.mark.parametrize("status", [BR.CONVERGED_S, BR.CONVERGED_R, BR.BREAKDOWN_DENOM, BR.BREAKDOWN_NONFINITE])
def test_frozen_state_makes_every_kernel_a_no_op(L, P, ws, status):
    vs = vectors(4)
    st = new_state(L, BR.SCALARS, status=status)
    before = snapshot(vs, st)
    for name in ("update_s", "dot2", "update_xr", "update_p"):
        run_kernel(L, name, vs, st, ws)
        assert unchanged(before, vs, st), f"{name} changed something in a frozen state"
    assert counter(ws, P) == 0


# ------------------------------------------------------------------------------------------ the solver
def make_sh(off, col, val, impl="b200"):
    from cudalibrarysamples_b200 import cusparse_api as cs
    from cudalibrarysamples_b200.sharded import ShardedCsr
    api = cs.Api(impl)

    def make_local(rr, cc, arrays):
        return cs.SpMVOperator(api, "csr", rr, cc, arrays, preprocess=True)
    return ShardedCsr(torch.from_numpy(off).cuda(), torch.from_numpy(col).cuda(), torch.from_numpy(val).cuda(), 0, 1, make_local,
                      balance="rows")


def bits(t):
    return t.view(torch.int64).clone()


def test_sample_system_converges_like_the_restatement_on_both_paths():
    from cudalibrarysamples_b200.bicgstab import FusedBicgstabSolver
    grid, tol = 700, 1e-10
    off, col, val = O.gen_stencil5(grid, 0.3, 0.3, 0.2)
    n = grid * grid
    A = sp.csr_matrix((val, col, off), shape=(n, n))
    b = 0.75 * (A @ np.ones(n))
    want = BR.fused(lambda v: A @ v, b, 2000, tol)
    sh = make_sh(off, col, val)
    try:
        bd = torch.from_numpy(b).cuda()
        runs = {}
        for graph in (True, False, True):
            solver = FusedBicgstabSolver(sh, bd, use_graph=graph)
            res = solver.run(2000, tol)
            runs.setdefault(graph, []).append((bits(res.x), res.status, res.iterations, res.history))
            if graph:
                # replays past the stop change nothing
                x_before, st_before = bits(solver.x), bits(solver.state)
                solver.replay(3)
                torch.cuda.synchronize()
                assert torch.equal(bits(solver.x), x_before) and torch.equal(bits(solver.state), st_before)
        (g1, g2), (e,) = runs[True], runs[False]
        assert torch.equal(g1[0], g2[0]) and g1[1:] == g2[1:], "two graph runs differ"
        assert torch.equal(g1[0], e[0]) and g1[1:] == e[1:], "graph and plain launches differ"
        _, status, iters, hist = g1
        # BiCGStab amplifies rounding (summation order, fused multiply-adds) from iteration to iteration on this non-normal
        # operator: on an H100 the relative gap to the numpy restatement grows from 1e-14 at the start to 1e-2 near the
        # threshold, and the GPU stops converged at r after 49 iterations where the restatement stops converged at s after 51
        # (its ||r_50|| is 1.07 threshold).  So the stop is checked to within 2 iterations, and the history to 1e-5 over the
        # first 25 iterations, where ||r|| is still far above the threshold (measured there: at most 1.7e-6).
        assert status in ("converged_s", "converged_r") and BR.STATUS_NAMES[want["status"]] in ("converged_s", "converged_r")
        assert abs(iters - want["iterations"]) <= 2, (iters, want["iterations"])
        h, w = np.asarray(hist[:26]), np.asarray(want["history"][:26])
        rel = np.abs(h - w) / w
        assert np.all(rel <= 1e-5), rel.tolist()
        thr = tol * want["history"][0]
        x = g1[0].view(torch.float64).cpu().numpy()
        assert np.linalg.norm(b - A @ x) < 10 * thr
    finally:
        sh.close()          # a failed assertion must not leave the operator to be freed during a later capture


def test_skew_symmetric_system_breaks_down_at_the_first_denominator():
    from cudalibrarysamples_b200.bicgstab import FusedBicgstabSolver
    n = 4096
    A = sp.diags([np.ones(n - 1), -np.ones(n - 1)], [1, -1], format="csr")
    A.sort_indices()
    b = E.nonzero_ints(np.random.default_rng(5), n, 1, 5).astype(np.float64)
    sh = make_sh(A.indptr.astype(np.int32), A.indices.astype(np.int32), A.data.astype(np.float64))
    for graph in (True, False):
        res = FusedBicgstabSolver(sh, torch.from_numpy(b).cuda(), use_graph=graph).run(50, 1e-10)
        assert res.status == "breakdown_denom" and res.iterations == 0
        assert not torch.any(res.x != 0) and not torch.any(torch.isnan(res.x))
    sh.close()


def test_dominant_nonsymmetric_rmat_converges_to_spsolve():
    from cudalibrarysamples_b200.bicgstab import FusedBicgstabSolver
    n = 20000
    off, col, val = O.rmat_csr(n, avg_nnz=8, seed=21, val_seed=22)
    R = sp.csr_matrix((val - 0.5, col, off), shape=(n, n))
    A = (R + sp.diags(np.abs(R).sum(axis=1).A1 + 1.0)).tocsr()
    A.sort_indices()
    b = O.uniform(23, n) - 0.5
    sh = make_sh(A.indptr.astype(np.int32), A.indices.astype(np.int32), A.data.astype(np.float64))
    res = FusedBicgstabSolver(sh, torch.from_numpy(b).cuda()).run(500, 1e-12)
    assert res.status in ("converged_s", "converged_r")
    ref = spla.spsolve(A.tocsc(), b)
    x = res.x.cpu().numpy()
    assert np.linalg.norm(x - ref) <= 1e-9 * np.linalg.norm(ref)
    assert np.linalg.norm(b - A @ x) <= 10 * 1e-12 * np.linalg.norm(b)
    sh.close()
