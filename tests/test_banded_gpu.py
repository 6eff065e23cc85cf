"""GPU: the batched banded solves of batched_banded.cu (DESIGN.md 3.25).

* The native C ABI, four value types x {gpsv, gtsv algo 0 / 1 / 2}, m up to 4096 and batch from 1 to 64K + 37: the backward error
  ||b - A x|| / (||A|| ||x||) within c m eps per system, the forward error against scipy's fp64 / complex128 solve, the coefficient
  arrays bitwise unchanged, canaries around x and the workspace intact, and two runs and a CUDA-graph replay bit-identical.
  Diagonally dominant systems, and well-conditioned ones with zero or tiny main-diagonal entries (gpsv and gtsv algo 1 / 2 only).
* The shim with B200SPMV_BANDED=on against the closed library on the same inputs, with the native / forwarded counts, the statuses
  the closed library gives for m < 3 and batch < 1 (forwarded, so the shim gives the same), and what the closed library leaves in
  the coefficient arrays (printed, not asserted).
* The unmodified cuSPARSE/gpsvInterleavedBatch sample linked against the closed library and against the shim."""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pytest
import scipy.linalg
import torch

from oracle import banded_ref as R

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DTYPES = [torch.float32, torch.float64, torch.complex64, torch.complex128]
VT = {torch.float32: 0, torch.float64: 1, torch.complex64: 4, torch.complex128: 5}
# (name, P, algo, W: our factor entries per row)
METHODS = [("gpsv", 2, 0, 4), ("gtsv0", 1, 0, 1), ("gtsv1", 1, 1, 2), ("gtsv2", 1, 2, 2)]
CANARY = 0x5C
PAD = 256


@pytest.fixture(scope="module")
def L():
    if not torch.cuda.is_available():
        pytest.skip("no GPU")
    from cudalibrarysamples_b200 import lib
    return lib.shim()


def stream():
    return torch.cuda.current_stream().cuda_stream


def eps(dt):
    return torch.finfo(torch.empty(0, dtype=dt).real.dtype).eps


def systems(m, batch, P, dt, seed, kind="dominant"):
    """(diags, b) as (m, batch) device tensors; out-of-band slots NaN.  kind as in tests/test_banded_cpu.py: diagonally dominant, or
    every other main-diagonal entry zero (gpsv) / 1e-30 (gtsv) with order-one off-diagonals."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    rdt = torch.float32 if dt in (torch.float32, torch.complex64) else torch.float64

    def draw():
        v = torch.rand(m, batch, device="cuda", generator=g, dtype=rdt) * 2 - 1
        if dt.is_complex:
            v = torch.complex(v, torch.rand(m, batch, device="cuda", generator=g, dtype=rdt) * 2 - 1)
        return v.to(dt)

    diags = [draw() for _ in range(2 * P + 1)]
    if kind == "dominant":
        diags[P] = diags[P] + torch.where(diags[P].real >= -0.5, 1.0, -1.0).to(dt) * (2 * P + 1.0)
    else:
        diags[P][::2] = diags[P][::2] * 1e-30 if P == 1 else 0
        for o in range(2 * P + 1):
            if o != P:
                diags[o] = diags[o] + torch.where(diags[o].real >= -1e-3, 1.0, -1.0).to(dt)
    mask = torch.tensor(R.band_mask(m, P), device="cuda")
    diags = [torch.where(mask[o][:, None], d, torch.full_like(d, float("nan"))).contiguous() for o, d in enumerate(diags)]
    return diags, draw().contiguous()


def backward_error(diags, x, b):
    """per system ||b - A x||_inf / (||A||_inf ||x||_inf), in complex128 on the device"""
    P = (len(diags) - 1) // 2
    m = x.shape[0]
    mask = torch.tensor(R.band_mask(m, P), device="cuda")
    xc = x.to(torch.complex128)
    Ax = torch.zeros_like(xc)
    rowsum = torch.zeros(x.shape, dtype=torch.float64, device="cuda")
    for o, d in enumerate(diags):
        dd = torch.where(mask[o][:, None], d.to(torch.complex128), 0)
        s = o - P                                           # row i reads x[i + s]
        lo, hi = max(0, -s), min(m, m - s)
        Ax[lo:hi] += dd[lo:hi] * xc[lo + s:hi + s]
        rowsum += dd.abs()
    r = (b.to(torch.complex128) - Ax).abs().amax(0)
    return (r / (rowsum.amax(0) * xc.abs().amax(0)).clamp_min(1e-300)).cpu().numpy()


def forward_error(diags, x, b, P, js):
    """max over systems js of ||x - x_scipy||_inf / ||x_scipy||_inf, scipy solving in complex128"""
    dn = [d.cpu().numpy() for d in diags]
    xn, bn = x.cpu().numpy(), b.cpu().numpy()
    worst = 0.0
    for j in js:
        want = scipy.linalg.solve_banded((P, P), R.banded_ab(dn, j).astype(np.complex128), bn[:, j].astype(np.complex128))
        worst = max(worst, np.abs(xn[:, j] - want).max() / max(np.abs(want).max(), 1e-300))
    return worst


def padded(n_bytes, dev="cuda"):
    """a canary-filled uint8 tensor with n_bytes in the middle, 256-byte aligned (PAD on either side)"""
    t = torch.full((n_bytes + 2 * PAD,), CANARY, dtype=torch.uint8, device=dev)
    return t, t[PAD:PAD + n_bytes]


def native_solve(L, name, P, algo, diags, x, work):
    dt = x.dtype
    m, batch = x.shape
    if P == 2:
        return L.b200gpsv_interleaved(stream(), VT[dt], m, *[d.data_ptr() for d in diags], x.data_ptr(), batch, work.data_ptr())
    return L.b200gtsv_interleaved(stream(), VT[dt], algo, m, *[d.data_ptr() for d in diags], x.data_ptr(), batch, work.data_ptr())


def ws_bytes(L, P, algo, dt, m, batch):
    return (L.b200gpsv_interleaved_workspace_bytes(VT[dt], m, batch) if P == 2 else
            L.b200gtsv_interleaved_workspace_bytes(VT[dt], algo, m, batch))


SHAPES = [(3, 1), (4, 65573), (5, 33), (32, 1000), (33, 4099), (257, 129), (1024, 64), (4096, 300)]


@pytest.mark.parametrize("name,P,algo,W", METHODS)
@pytest.mark.parametrize("dt", DTYPES)
def test_native_solves_dominant_systems(L, name, P, algo, W, dt):
    for m, batch in SHAPES:
        diags, b = systems(m, batch, P, dt, seed=m * 7 + batch)
        before = [d.clone() for d in diags]
        w = torch.empty(0, dtype=dt).element_size()
        xbuf, xb = padded(m * batch * w)
        x = xb.view(dt).view(m, batch)
        x.copy_(b)
        need = ws_bytes(L, P, algo, dt, m, batch)
        assert need == W * m * batch * w
        wbuf, work = padded(need)
        assert native_solve(L, name, P, algo, diags, x, work) == 0
        torch.cuda.synchronize()
        assert torch.isfinite(torch.view_as_real(x) if dt.is_complex else x).all(), (m, batch)
        be = backward_error(diags, x, b)
        assert be.max() <= 8 * m * eps(dt), (m, batch, be.max())
        js = sorted({0, batch - 1, batch // 2, batch // 3})
        fe = forward_error(diags, x, b, P, js)
        assert fe <= 50 * m * eps(dt), (m, batch, fe)
        for d0, d1 in zip(before, diags):                     # the coefficients, NaN slots included, bit for bit
            assert torch.equal(d0.view(torch.uint8), d1.view(torch.uint8))
        for buf in (xbuf, wbuf):
            assert (buf[:PAD] == CANARY).all() and (buf[-PAD:] == CANARY).all(), (m, batch)


@pytest.mark.parametrize("name,P,algo,W", [m for m in METHODS if m[0] != "gtsv0"])
@pytest.mark.parametrize("dt", DTYPES)
def test_native_solves_zero_and_tiny_pivots(L, name, P, algo, W, dt):
    """algo 0 is not required to solve these; gpsv and gtsv algo 1 / 2 must"""
    for m, batch in ((4, 5), (64, 1000), (1024, 70)):
        diags, b = systems(m, batch, P, dt, seed=m, kind="zero_diag")
        x = b.clone()
        work = torch.empty(ws_bytes(L, P, algo, dt, m, batch), dtype=torch.uint8, device="cuda")
        assert native_solve(L, name, P, algo, diags, x, work) == 0
        torch.cuda.synchronize()
        be = backward_error(diags, x, b)
        assert np.isfinite(be).all() and be.max() <= 8 * m * eps(dt), (m, be.max())



# subnormal magnitudes: below the smallest normal number (fp32 1.2e-38, fp64 2.2e-308), so 1 / |d| overflows
TINY = {torch.float32: 1e-40, torch.complex64: 1e-40, torch.float64: 1e-310, torch.complex128: 1e-310}


@pytest.mark.parametrize("name,P,algo,W", [m for m in METHODS if m[0] != "gtsv0"])
@pytest.mark.parametrize("dt", DTYPES)
def test_native_solves_subnormal_pivots(L, name, P, algo, W, dt):
    """Well-conditioned systems with subnormal main-diagonal entries, against scipy on the same inputs: the 4 x 4 system
    d = (tiny, 3, 3, 3) with off-diagonals 1 (condition number about 13), then 4099 systems of 64 rows whose every other
    main-diagonal entry is subnormal."""
    tiny = TINY[dt]
    cases = []
    d4 = [torch.full((4, 1), 1.0 if abs(o - P) == 1 else 0.5, dtype=torch.float64) for o in range(2 * P + 1)]
    d4[P] = torch.tensor([[tiny], [3.0], [3.0], [3.0]], dtype=torch.float64)
    cases.append(([d.to(dt).cuda() for d in d4], torch.arange(1.0, 5.0, dtype=torch.float64)[:, None].to(dt).cuda()))
    diags, b = systems(64, 4099, P, dt, seed=11, kind="zero_diag")
    diags[P][::2] = torch.where(diags[P][::2].real >= 0, 1.0, -1.0).to(dt) * torch.tensor(tiny, dtype=torch.float64).to(dt)
    cases.append((diags, b))
    for diags, b in cases:
        m, batch = b.shape
        assert (diags[P][0].abs() < torch.finfo(torch.empty(0, dtype=dt).real.dtype).tiny).all() and (diags[P][0] != 0).all()
        x = b.clone()
        work = torch.empty(ws_bytes(L, P, algo, dt, m, batch), dtype=torch.uint8, device="cuda")
        assert native_solve(L, name, P, algo, diags, x, work) == 0
        torch.cuda.synchronize()
        assert torch.isfinite(torch.view_as_real(x) if dt.is_complex else x).all(), m
        dn = [d.cpu().numpy() for d in diags]
        xn, bn = x.cpu().numpy(), b.cpu().numpy()
        for j in sorted({0, 1, batch // 2, batch - 1} & set(range(batch))):
            want = scipy.linalg.solve_banded((P, P), R.banded_ab(dn, j).astype(np.complex128), bn[:, j].astype(np.complex128))
            cond = np.linalg.cond(R.dense(dn, j).astype(np.complex128))
            assert np.abs(xn[:, j] - want).max() <= 100 * m * eps(dt) * cond * np.abs(want).max(), (m, j, cond)

@pytest.mark.parametrize("name,P,algo,W", METHODS)
@pytest.mark.parametrize("dt", [torch.float32, torch.complex128])
def test_runs_and_graph_replay_are_bit_identical(L, name, P, algo, W, dt):
    m, batch = 200, 3000
    diags, b = systems(m, batch, P, dt, seed=3)
    work = torch.full((ws_bytes(L, P, algo, dt, m, batch),), 0x7F, dtype=torch.uint8, device="cuda")
    outs = []
    for _ in range(2):
        x = b.clone()
        assert native_solve(L, name, P, algo, diags, x, work) == 0
        torch.cuda.synchronize()
        outs.append(x)
        work.fill_(0xA5)                                       # a stale workspace changes nothing
    x = b.clone()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    g = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s):
        with torch.cuda.graph(g, stream=s):
            x.copy_(b)
            assert native_solve(L, name, P, algo, diags, x, work) == 0
    torch.cuda.current_stream().wait_stream(s)
    for _ in range(2):
        x.fill_(0)
        g.replay()
        torch.cuda.synchronize()
        outs.append(x.clone())
    for o in outs[1:]:
        assert torch.equal(o.view(torch.uint8), outs[0].view(torch.uint8))


# ---- through the shim, against the closed library -------------------------------------------------------------------------------
@pytest.fixture()
def api_pair(L):
    from cudalibrarysamples_b200 import cusparse_api as cs
    ours, closed = cs.Api("b200"), cs.Api("cusparse")
    ours.set_option("B200SPMV_BANDED", "on")
    yield cs, ours, closed
    ours.set_option("B200SPMV_BANDED", "auto")


def _shim_solve(cs, api, P, algo, diags, x):
    return cs.gpsv_interleaved(api, *diags, x, algo) if P == 2 else cs.gtsv_interleaved(api, *diags, x, algo)


@pytest.mark.parametrize("name,P,algo,W", METHODS)
@pytest.mark.parametrize("dt", DTYPES)
def test_shim_native_against_the_closed_library(api_pair, name, P, algo, W, dt):
    cs, ours, closed = api_pair
    for m, batch in ((4, 2), (77, 1030), (1024, 256)):
        diags, b = systems(m, batch, P, dt, seed=m + P)
        diags = [torch.nan_to_num(d, nan=0.0) for d in diags]          # the closed library's out-of-band handling is its own
        before = [d.clone() for d in diags]
        ours.reset_stats()
        xo = _shim_solve(cs, ours, P, algo, diags, b.clone())
        st = ours.stats()
        assert st["native"] == 1 and st["forwarded"] == 0, st
        for d0, d1 in zip(before, diags):
            assert torch.equal(d0.view(torch.uint8), d1.view(torch.uint8))
        cd = [d.clone() for d in diags]
        xc = _shim_solve(cs, closed, P, algo, cd, b.clone())
        changed = [i for i, (d0, d1) in enumerate(zip(before, cd)) if not torch.equal(d0.view(torch.uint8), d1.view(torch.uint8))]
        print(f"closed {name} {dt} m={m} batch={batch}: coefficient arrays written: {changed} (0 = first sub-diagonal passed)")
        for x in (xo, xc):
            assert backward_error(diags, x, b).max() <= 8 * m * eps(dt), (m, batch)
        assert ((xo - xc).abs().amax(0) <= 100 * m * eps(dt) * xc.abs().amax(0)).all(), (m, batch)


def test_shim_default_route_follows_the_measured_table(L):
    from cudalibrarysamples_b200 import cusparse_api as cs
    api = cs.Api("b200")
    diags, b = systems(64, 64, 1, torch.float64, seed=1)
    diags = [torch.nan_to_num(d, nan=0.0) for d in diags]
    api.reset_stats()
    cs.gtsv_interleaved(api, *diags, b.clone(), 1)
    from scripts.banded_bench import native
    want = int(native(1, 1, 1, 64, 64))
    assert api.stats()["native"] == want and api.stats()["forwarded"] == 1 - want


def test_closed_statuses_for_small_and_empty_sizes_are_kept(api_pair):
    """m < 3 and batch < 1 are forwarded, so the shim gives whatever the closed library gives; printed for DESIGN.md 3.25"""
    cs, ours, closed = api_pair
    R_ = closed.real
    arrays = torch.zeros(6, 64, dtype=torch.float32, device="cuda")          # room for every m x batch tried below
    ptrs = [C.c_void_p(a.data_ptr()) for a in arrays]
    h = closed.cusparseCreate()
    try:
        for m, batch in ((0, 4), (1, 4), (2, 4), (3, 4), (4, 0), (4, -1), (-1, 4)):
            for op, n in (("gpsv", 5), ("gtsv", 3)):
                for algo in ((0, 1) if op == "gpsv" else (0, 1, 2, 3)):
                    got = []
                    for lib in (R_, ours.lib):
                        size = C.c_size_t(0)
                        s1 = getattr(lib, f"cusparseS{op}InterleavedBatch_bufferSizeExt")(h, algo, m, *ptrs[:n + 1], batch, C.byref(size))
                        s2 = None
                        if s1 == 0 and m >= 0 and batch >= 1:          # solve only with the workspace the library asked for
                            work = torch.empty(max(size.value, 16), dtype=torch.uint8, device="cuda")
                            s2 = getattr(lib, f"cusparseS{op}InterleavedBatch")(h, algo, m, *ptrs[:n + 1], batch, C.c_void_p(work.data_ptr()))
                            torch.cuda.synchronize()
                        got.append((s1, s2))
                    print(f"closed S{op} algo={algo} m={m} batch={batch}: bufferSizeExt {got[0][0]}, solve {got[0][1]}")
                    assert got[0] == got[1], (op, algo, m, batch, got)
    finally:
        closed.cusparseDestroy(h)


def test_reference_sample_on_both_libraries(L):
    exes = [os.path.join(ROOT, "oracle", "_ref", f"gpsvInterleavedBatch_example.{k}") for k in ("cusparse", "b200")]
    if not all(os.path.exists(e) for e in exes):
        pytest.skip("oracle/_ref not built (needs the reference checkout at build time)")
    outs = []
    for exe, env in ((exes[0], {}), (exes[1], {"B200SPMV_LOG": "1", "B200SPMV_BANDED": "on"})):
        p = subprocess.run([exe], capture_output=True, text=True, env=dict(os.environ, **env), timeout=300)
        assert p.returncode == 0, p.stdout + p.stderr
        outs.append(p)
        print(p.stdout)
    xs = [re.findall(r"x\d\[\d\] = (\S+)", p.stdout) for p in outs]
    assert len(xs[0]) == 8 and xs[0] == xs[1], xs
    G = R.sample()
    assert np.allclose([float(v) for v in xs[1]], G["x"], atol=1e-6)
    for p in outs:
        res = [float(v) for v in re.findall(r"\| = (\S+)", p.stdout)]
        assert len(res) == 2 and max(res) <= 1e-5, res
    assert re.search(r"\[b200spmv\] SgpsvInterleavedBatch native", outs[1].stderr), outs[1].stderr
