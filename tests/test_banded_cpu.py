"""CPU: the batched banded solves (batched_banded.cuh / .cu, DESIGN.md 3.25) without a GPU.

* oracle/banded_ref.py's Givens / pivoted-LU / Thomas steps against scipy.linalg.solve_banded, and against the sample's golden arrays;
* the kernels' OWN SOURCE compiled for the host on tests/host_emulation/cuda_emulation.h (a real thread per lane) against that
  restatement, for the four value types, sizes around the warp width and batch counts that leave the last CTA partial;
* NaN in the out-of-band slots never reaches x; the coefficient arrays are left as they were;
* the workspace formulas, host-side argument rejection, b200banded_route's table with and without B200SPMV_FORWARD, and the
  exported symbols."""
import ctypes as C
import os
import subprocess
import sys
import textwrap

import numpy as np
import pytest
import scipy.linalg

from oracle import banded_ref as R
from test_abi import declared_symbols, exported

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMU_DIR = os.path.join(ROOT, "tests", "host_emulation")
REAL = "/usr/local/cuda/lib64/libcusparse.so.12"
DTYPES = [np.float32, np.float64, np.complex64, np.complex128]
EMU_VT = {np.float32: 0, np.float64: 1, np.complex64: 2, np.complex128: 3}
CUDA_VT = {np.float32: 0, np.float64: 1, np.complex64: 4, np.complex128: 5}
# (name, P, oracle method, emulation method, W)
METHODS = [("gpsv", 2, R.GIVENS, 0, 4), ("gtsv0", 1, R.THOMAS, 1, 1), ("gtsv1", 1, R.PIVOT_LU, 2, 2), ("gtsv2", 1, R.GIVENS, 3, 2)]
NEW = ["b200gpsv_interleaved", "b200gpsv_interleaved_workspace_bytes", "b200gtsv_interleaved", "b200gtsv_interleaved_workspace_bytes",
       "b200banded_route"] + [f"cusparse{t}{op}InterleavedBatch{s}" for t in "SDCZ" for op in ("gpsv", "gtsv") for s in ("", "_bufferSizeExt")]


def systems(m, batch, P, dtype, seed, kind="dominant"):
    """(diags, b) interleaved (m, batch).  dominant: |d| > sum of the off-diagonals.  zero_diag: every other main-diagonal entry
    zero or tiny, the off-diagonals of order one -- well conditioned, but a pivot-free elimination meets a zero pivot.  The
    out-of-band slots hold NaN."""
    rng = np.random.default_rng(seed)

    def draw(scale=1.0):
        v = rng.uniform(-1, 1, (m, batch)) * scale
        if np.iscomplexobj(np.zeros(0, dtype)):
            v = v + 1j * rng.uniform(-1, 1, (m, batch)) * scale
        return v

    diags = [draw() for _ in range(2 * P + 1)]
    if kind == "dominant":
        diags[P] = diags[P] + np.sign(diags[P].real + 0.5) * (2 * P + 1.0)
    else:
        diags[P][::2] = 1e-30 * diags[P][::2] if P == 1 else 0
        for o in range(2 * P + 1):
            if o != P:
                diags[o] = diags[o] + np.sign(diags[o].real + 1e-3) * 1.0
    mask = R.band_mask(m, P)
    diags = [np.where(mask[o][:, None], d, np.nan).astype(dtype) for o, d in enumerate(diags)]
    return diags, draw().astype(dtype)


def _tol(dtype):
    return 200 * np.finfo(np.zeros(0, dtype).real.dtype).eps


# ---- the restatement --------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name,P,method,_e,_w", METHODS)
@pytest.mark.parametrize("dtype", [np.float64, np.complex128])
@pytest.mark.parametrize("kind", ["dominant", "zero_diag"])
def test_restatement_matches_solve_banded(name, P, method, _e, _w, dtype, kind):
    if kind == "zero_diag" and method == R.THOMAS:
        pytest.skip("Thomas without pivoting is not required to solve a system with zero pivots")
    for m in (3, 4, 5, 31, 33):
        diags, b = systems(m, 3, P, dtype, seed=m + 10 * P, kind=kind)
        x = R.solve(diags, b, method)
        for j in range(3):
            want = scipy.linalg.solve_banded((P, P), R.banded_ab(diags, j), b[:, j].astype(np.complex128))
            cond = np.linalg.cond(R.dense(diags, j))
            assert np.abs(x[:, j] - want).max() <= 1e-14 * m * cond * np.abs(want).max(), (m, j, cond)
        assert R.backward_error(diags, x, b).max() <= 4 * m * np.finfo(np.float64).eps


def test_restatement_reproduces_the_sample():
    G = R.sample()
    m, batch = G["m"], G["batch"]
    inter = lambda v: np.array(v, np.float32).reshape(batch, m).T         # noqa: E731
    diags = [inter(G[k]) for k in ("ds", "dl", "d", "du", "dw")]
    x = R.solve(diags, inter(G["b"]), R.GIVENS)
    assert np.allclose(x.T.reshape(-1), G["x"], rtol=1e-5, atol=1e-6)
    assert np.round(x.T.reshape(-1).astype(np.float64), 4).tolist() == G["x_printed"]


# ---- the kernels' own source on the host ---------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def emu():
    out = os.path.join(EMU_DIR, "_build", "libbanded_emu.so")
    srcs = [os.path.join(EMU_DIR, "emulate_banded.cpp"), os.path.join(EMU_DIR, "cuda_emulation.h"),
            os.path.join(ROOT, "cudalibrarysamples_b200", "csrc", "batched_banded.cuh")]
    if not os.path.exists(out) or any(os.path.getmtime(s) > os.path.getmtime(out) for s in srcs):
        os.makedirs(os.path.dirname(out), exist_ok=True)
        subprocess.check_call(["g++", "-O1", "-std=c++17", "-pthread", "-shared", "-fPIC", "-I" + EMU_DIR,
                               "-I" + os.path.join(ROOT, "cudalibrarysamples_b200", "csrc"), srcs[0], "-o", out])
    return C.CDLL(out)


def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def run_emu(emu, e, P, W, diags, b):
    m, batch = b.shape
    x = b.copy()
    work = np.full((W * m, batch), np.nan, b.dtype)
    d = [None] * (2 - P) + diags + [None] * (2 - P)
    assert emu.emu_banded(e, EMU_VT[b.dtype.type], C.c_longlong(m), C.c_longlong(batch), *map(_p, d), _p(x), _p(work)) == 0
    return x


@pytest.mark.parametrize("name,P,method,e,W", METHODS)
@pytest.mark.parametrize("dtype", DTYPES)
def test_kernel_source_matches_the_restatement(emu, name, P, method, e, W, dtype):
    """Same steps in the same order: fp64 / complex128 agree to the last bits, fp32 / complex64 within a few ulps of the answer."""
    for m, batch in ((3, 33), (4, 1), (5, 70), (31, 37), (32, 5), (33, 129), (257, 3)):
        diags, b = systems(m, batch, P, dtype, seed=1000 + m)
        before = [d.copy() for d in diags]
        x = run_emu(emu, e, P, W, diags, b)
        want = R.solve(diags, b, method)
        scale = np.abs(want).max(axis=0)
        assert (np.abs(x - want).max(axis=0) <= 8 * np.finfo(np.zeros(0, dtype).real.dtype).eps * m * scale).all(), (m, batch)
        assert R.backward_error(diags, x, b).max() <= _tol(dtype) * m, (m, batch)
        for d0, d1 in zip(before, diags):                       # the coefficients (NaN slots included) are left as they were
            assert d0.tobytes() == d1.tobytes()


@pytest.mark.parametrize("name,P,method,e,W", [m for m in METHODS if m[2] != R.THOMAS])
@pytest.mark.parametrize("dtype", [np.float32, np.complex128])
def test_kernel_source_solves_zero_and_tiny_pivots(emu, name, P, method, e, W, dtype):
    m, batch = 34, 40                                            # even: with every other diagonal entry 0, an odd m is singular
    diags, b = systems(m, batch, P, dtype, seed=7, kind="zero_diag")
    x = run_emu(emu, e, P, W, diags, b)
    assert np.isfinite(x).all()
    assert R.backward_error(diags, x, b).max() <= _tol(dtype) * m


@pytest.mark.parametrize("name,P,method,e,W", METHODS)
def test_out_of_band_nan_never_reaches_x(emu, name, P, method, e, W):
    """systems() already puts NaN in every out-of-band slot; here also Inf, and m = 3, where those slots are a large share."""
    for m in (3, 4, 6):
        diags, b = systems(m, 65, P, np.float64, seed=m)
        mask = R.band_mask(m, P)
        for o, d in enumerate(diags):
            d[~mask[o], 1::2] = np.inf
        x = run_emu(emu, e, P, W, diags, b)
        assert np.isfinite(x).all()
        assert R.backward_error(diags, x, b).max() <= _tol(np.float64) * m


def test_sample_on_the_kernel_source(emu):
    G = R.sample()
    m, batch = G["m"], G["batch"]
    inter = lambda v: np.ascontiguousarray(np.array(v, np.float32).reshape(batch, m).T)   # noqa: E731
    x = run_emu(emu, 0, 2, 4, [inter(G[k]) for k in ("ds", "dl", "d", "du", "dw")], inter(G["b"]))
    assert np.allclose(x.T.reshape(-1), G["x"], rtol=1e-5, atol=1e-6)
    assert np.round(x.T.reshape(-1).astype(np.float64), 4).tolist() == G["x_printed"]



# subnormal magnitudes: below the smallest normal number (fp32 1.2e-38, fp64 2.2e-308), so 1 / |d| overflows
TINY = {np.float32: 1e-40, np.complex64: 1e-40, np.float64: 1e-310, np.complex128: 1e-310}


def subnormal_cases(P, dtype):
    """(diags, b): the 4 x 4 system d = (tiny, 3, 3, 3) with off-diagonals 1 (condition number about 13), and 64 systems of 36
    rows whose every other main-diagonal entry is subnormal, with order-one off-diagonals."""
    tiny = TINY[dtype]
    m = 4
    diags = [np.full((m, 1), 1.0 if abs(o - P) == 1 else 0.5) for o in range(2 * P + 1)]
    diags[P] = np.array([[tiny], [3.0], [3.0], [3.0]])
    yield [d.astype(dtype) for d in diags], np.arange(1.0, m + 1)[:, None].astype(dtype)
    diags, b = systems(36, 64, P, dtype, seed=5, kind="zero_diag")
    diags[P][::2] = (np.sign(diags[P][::2].real + 0.5) * tiny).astype(dtype)
    yield diags, b


def assert_matches_a_dense_solve(diags, b, x):
    """x against scipy.linalg.solve_banded on the same (rounded) inputs in complex128, within 100 m eps cond"""
    P, m = (len(diags) - 1) // 2, b.shape[0]
    eps = np.finfo(np.zeros(0, b.dtype).real.dtype).eps
    assert np.isfinite(x).all()
    for j in range(b.shape[1]):
        want = scipy.linalg.solve_banded((P, P), R.banded_ab(diags, j).astype(np.complex128), b[:, j].astype(np.complex128))
        cond = np.linalg.cond(R.dense(diags, j).astype(np.complex128))
        assert np.abs(x[:, j] - want).max() <= 100 * m * eps * cond * np.abs(want).max(), (j, cond)


@pytest.mark.parametrize("name,P,method,e,W", [m for m in METHODS if m[2] != R.THOMAS])
@pytest.mark.parametrize("dtype", DTYPES)
def test_kernel_source_and_restatement_solve_subnormal_pivots(emu, name, P, method, e, W, dtype):
    """A subnormal main-diagonal entry in a well-conditioned system: the Givens phase top / |top| and every division by a pivot
    must not go through a reciprocal, which overflows to Inf there."""
    for diags, b in subnormal_cases(P, dtype):
        assert_matches_a_dense_solve(diags, b, run_emu(emu, e, P, W, diags, b))
        with np.errstate(all="ignore"):
            assert_matches_a_dense_solve(diags, b, R.solve(diags, b, method))

# ---- the library: symbols, workspace, argument rejection, route ---------------------------------------------------------------
def test_header_declares_and_library_exports_the_banded_symbols(built_lib):
    names = declared_symbols()
    have = exported(built_lib)
    for n in NEW:
        assert n in names and n in have, n


def test_workspace_formulas(built_lib):
    from cudalibrarysamples_b200.lib import load
    L = load(built_lib)
    for dt, w in ((np.float32, 4), (np.float64, 8), (np.complex64, 8), (np.complex128, 16)):
        vt = CUDA_VT[dt]
        for m, batch in ((3, 1), (4096, 65536), (1 << 20, 3000)):
            assert L.b200gpsv_interleaved_workspace_bytes(vt, m, batch) == 4 * m * batch * w
            for algo, W in ((0, 1), (1, 2), (2, 2)):
                assert L.b200gtsv_interleaved_workspace_bytes(vt, algo, m, batch) == W * m * batch * w
        assert L.b200gpsv_interleaved_workspace_bytes(vt, 0, 4) == 0 and L.b200gpsv_interleaved_workspace_bytes(vt, 4, 0) == 0
        assert L.b200gtsv_interleaved_workspace_bytes(vt, 3, 4, 4) == 0
    assert L.b200gpsv_interleaved_workspace_bytes(2, 4, 4) == 0          # CUDA_R_16F: not a type the solves take


def test_host_side_argument_rejection(built_lib):
    """-1 before any launch (so no device is touched): bad type, algo, size, NULL or misaligned pointers."""
    from cudalibrarysamples_b200.lib import load
    L = load(built_lib)
    buf = (C.c_double * 512)()
    a = C.addressof(buf) // 16 * 16 + 16
    p = [a] * 5
    assert L.b200gpsv_interleaved(None, 2, 4, *p, a, 4, a) == -1                          # CUDA_R_16F
    assert L.b200gpsv_interleaved(None, 0, 0, *p, a, 4, a) == -1                          # m = 0
    assert L.b200gpsv_interleaved(None, 0, 4, *p, a, 0, a) == -1                          # batch = 0
    assert L.b200gpsv_interleaved(None, 0, 1 << 31, *p, a, 4, a) == -1                    # m past INT32_MAX
    assert L.b200gpsv_interleaved(None, 0, 4, None, a, a, a, a, a, 4, a) == -1            # a NULL diagonal
    assert L.b200gpsv_interleaved(None, 0, 4, *p, a, 4, None) == -1                       # no workspace
    assert L.b200gpsv_interleaved(None, 0, 4, *p, a, 4, a + 4) == -1                      # a workspace not 16-byte aligned
    assert L.b200gpsv_interleaved(None, 1, 4, a + 4, a, a, a, a, a, 4, a) == -1           # fp64 diagonal on a 4-byte boundary
    assert L.b200gtsv_interleaved(None, 0, 3, 4, a, a, a, a, 4, a) == -1                  # algo 3
    assert L.b200gtsv_interleaved(None, 5, 1, 4, a, a, a, a + 8, 4, a) == -1              # complex128 x on an 8-byte boundary
    assert L.b200gtsv_interleaved(None, 0, -1, 4, a, a, a, a, 4, a) == -1


ROUTE = textwrap.dedent(r"""
    import ctypes as C, os, sys
    sys.path.insert(0, os.path.dirname(os.path.dirname(sys.argv[1])))     # the repository: argv[1] is its built library
    from cudalibrarysamples_b200.lib import load
    shim = load(sys.argv[1])
    forward = sys.argv[2] == "forward"
    from scripts.banded_bench import native
    if sys.argv[2] == "on":
        assert shim.b200spmv_set_option(b"B200SPMV_BANDED", b"on") == 0
        native = lambda *a: True
    assert shim.b200spmv_set_option(b"B200SPMV_BANDED", b"sometimes") == -1
    buf = (C.c_double * 64)()
    ok = C.addressof(buf) // 16 * 16 + 16
    GPSV, GTSV = 0, 1
    for vt in (0, 1, 4, 5):
        for m in (3, 4, 16, 63, 64, 100, 256, 1024, 4096, 4097, 1 << 20):
            for batch in (1, 2, 1000, 1024, 16384, 40000, 65536, 262144, 1048576, 1048577):
                for op, algos in ((GPSV, (0,)), (GTSV, (0, 1, 2))):
                    for algo in algos:
                        want = 0 if forward else int(native(op, vt, algo, m, batch))
                        assert shim.b200banded_route(op, vt, algo, m, batch, ok) == want, (op, vt, algo, m, batch)
                        assert shim.b200banded_route(op, vt, algo, m, batch, None) == 0
                        assert shim.b200banded_route(op, vt, algo, m, batch, ok + 8) == 0
        for m, batch in ((0, 4), (1, 4), (2, 4), (4, 0), (4, -1), ((1 << 31), 4), (4, (1 << 31))):   # the closed library's verdict
            for op, algo in ((GPSV, 0), (GTSV, 0), (GTSV, 1), (GTSV, 2)):
                assert shim.b200banded_route(op, vt, algo, m, batch, ok) == 0, (op, m, batch)
        assert shim.b200banded_route(GPSV, vt, 1, 64, 64, ok) == 0 and shim.b200banded_route(GTSV, vt, 3, 64, 64, ok) == 0
        assert shim.b200banded_route(GTSV, vt, -1, 64, 64, ok) == 0 and shim.b200banded_route(2, vt, 0, 64, 64, ok) == 0
    for vt in (2, 3, 6, 7, 14):                                            # 16-bit, integer and unknown types
        assert shim.b200banded_route(GPSV, vt, 0, 64, 64, ok) == 0 and shim.b200banded_route(GTSV, vt, 1, 64, 64, ok) == 0
    print("OK")
""")


@pytest.mark.parametrize("mode", ["default", "forward", "on"])
def test_route_table(built_lib, mode):
    if not os.path.exists(REAL):
        pytest.skip("no toolkit libcusparse here")
    env = {k: v for k, v in os.environ.items() if not k.startswith("B200SPMV_")}
    env["B200SPMV_CUSPARSE"] = REAL
    if mode == "forward":
        env["B200SPMV_FORWARD"] = "1"
    p = subprocess.run([sys.executable, "-c", ROUTE, built_lib, mode], capture_output=True, text=True, timeout=600, env=env)
    assert p.returncode == 0 and p.stdout.strip().endswith("OK"), p.stdout + p.stderr
