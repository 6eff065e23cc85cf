"""GPU: the incomplete LU / Cholesky factorizations of ilu0_csr.cu (cusparse<t>csrilu02 / csric02, DESIGN.md 3.26).

* The native C ABI bit for bit against oracle/ilu0_ref.py in fp32 and fp64: 5-point stencils of both samples, the bidiagonal chain,
  the diagonal, a diagonally dominant R-MAT, base 0 and 1, rows that store both triangles.  The IC upper triangle is bitwise
  unchanged, canaries around the values and the workspace stay intact, and two factorizations give the same bits.
* Zero pivots on the native ABI: an ILU pivot that cancels (with and without boost, host and device scalars), IC pivots that are
  zero or negative.
* The shim with B200SPMV_ILU0=on against the closed library on the 700^2 sample matrices, and the statuses and positions of
  cusparseX*_zeroPivot after analysis and after the factorization, host and device pointer mode, pinned against the closed library.
* The unmodified cg and bicgstab samples with native SpSV, with B200SPMV_ILU0=on: the factorization runs natively and the solvers
  converge as the golden trace says."""
import ctypes as C
import json
import os
import subprocess

import numpy as np
import pytest
import torch

from oracle import ilu0_ref as R
from oracle import oracle as O

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NP = {torch.float32: np.float32, torch.float64: np.float64}
DT = {torch.float32: 0, torch.float64: 1}
KIND = {"lu": 0, "ic": 1}
CANARY = 0x5C
PAD = 256


@pytest.fixture(scope="module")
def L():
    if not torch.cuda.is_available():
        pytest.skip("no GPU")
    from cudalibrarysamples_b200 import lib
    return lib.shim()


@pytest.fixture(scope="module")
def cs():
    from cudalibrarysamples_b200 import cusparse_api
    return cusparse_api


def stream():
    return torch.cuda.current_stream().cuda_stream


_CASES = {}


def case(name, dtype):
    """(off, col, values, base 0) of a named test matrix, values in dtype."""
    key = (name, dtype)
    if key not in _CASES:
        if name == "cg100":
            off, col, val = O.gen_stencil5(100)
        elif name == "bicgstab100":
            off, col, val = O.gen_stencil5(100, mass=0.3, ux=0.3, uy=0.2)
        elif name == "chain":
            off, col = R.chain(1 << 12)
            val = R.dominant(off, col, np.float64, 3)
        elif name == "diagonal":
            off, col = R.diagonal(1 << 16)
            val = np.linspace(0.5, 4.0, 1 << 16)
        elif name == "rmat":
            off, col, _ = O.rmat_csr(20000, avg_nnz=8, seed=11, val_seed=12)
            off, col = R.with_diagonal(off, col, 20000)
            val = R.dominant(off, col, np.float64, 13)
        else:
            raise KeyError(name)
        _CASES[key] = (np.asarray(off, np.int32), np.asarray(col, np.int32), np.asarray(val).astype(NP[dtype]))
    return _CASES[key]


def native(L, kind, off, col, val, base, boost=None, on_device=False, runs=1):
    """analysis + `runs` factorizations from the same input on the native ABI, with canaries around the values and behind the
    workspace.  Returns (values after each run, structural zero, levels, zero-pivot position)."""
    rows, nnz = off.size - 1, col.size
    dt = torch.float32 if val.dtype == np.float32 else torch.float64
    offd, cold = torch.tensor(off + base, device="cuda"), torch.tensor(col + base, device="cuda")
    wsb = L.b200ilu0_workspace_bytes(rows, nnz)
    ws = torch.full((wsb + PAD,), CANARY, dtype=torch.uint8, device="cuda")
    sz, lev = C.c_int64(-9), C.c_int64(-9)
    assert L.b200ilu0_analysis(stream(), rows, nnz, offd.data_ptr(), cold.data_ptr(), base, ws.data_ptr(), C.byref(sz), C.byref(lev)) == 0
    outs = []
    for _ in range(runs):
        buf = torch.full((nnz + 2 * PAD,), float("nan"), dtype=dt, device="cuda")
        canary = buf.clone()
        v = buf[PAD:PAD + nnz]
        v.copy_(torch.tensor(val, device="cuda"))
        args = (0, None, None, 0)
        keep = None
        if boost is not None:
            tol, bval = boost
            if on_device:
                keep = (torch.tensor([tol], dtype=torch.float64, device="cuda"), torch.tensor([bval], dtype=dt, device="cuda"))
                args = (1, keep[0].data_ptr(), keep[1].data_ptr(), 1)
            else:
                keep = (C.c_double(tol), (C.c_float if dt == torch.float32 else C.c_double)(bval))
                args = (1, C.addressof(keep[0]), C.addressof(keep[1]), 0)
        rc = L.b200ilu0_factor(stream(), KIND[kind], DT[dt], rows, nnz, offd.data_ptr(), cold.data_ptr(), base, v.data_ptr(), *args,
                               ws.data_ptr())
        torch.cuda.synchronize()
        assert rc == 0
        both = torch.cat([buf[:PAD], buf[PAD + nnz:]])
        assert torch.isnan(both).all() and both.numel() == 2 * PAD, "canary around the values overwritten"
        del canary
        outs.append(v.cpu().numpy().copy())
    assert (ws[wsb:] == CANARY).all(), "canary behind the workspace overwritten"
    assert np.array_equal(offd.cpu().numpy(), off + base) and np.array_equal(cold.cpu().numpy(), col + base)
    pos = C.c_int(-7)
    assert L.b200ilu0_zero_pivot(stream(), ws.data_ptr(), C.byref(pos), 0, None) == 0
    return outs, sz.value, lev.value, pos.value


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
@pytest.mark.parametrize("kind", ["lu", "ic"])
@pytest.mark.parametrize("name", ["cg100", "bicgstab100", "chain", "diagonal", "rmat"])
def test_native_factor_is_the_oracle_bit_for_bit(L, name, kind, dtype):
    off, col, val = case(name, dtype)
    for base in (0, 1):
        outs, sz, lev, pos = native(L, kind, off, col, val, base, runs=2 if base == 0 else 1)
        want, wpos = R.factor(kind, off + base, col + base, val, base)
        assert sz == -1 and lev == R.levels(off, col).max() + 1
        assert np.array_equal(outs[0].view(np.uint8), want.view(np.uint8)), (name, kind, base)
        assert pos == wpos == -1
        if len(outs) > 1:
            assert np.array_equal(outs[0].view(np.uint8), outs[1].view(np.uint8))
        if kind == "ic":                     # rows that store both triangles: the upper one is untouched
            rowof = np.repeat(np.arange(off.size - 1), np.diff(off))
            up = col > rowof
            assert np.array_equal(outs[0][up].view(np.uint8), val[up].view(np.uint8))


def small(dense):
    A = np.asarray(dense, np.float64)
    rows, cols = np.nonzero(A)
    off = np.concatenate([[0], np.cumsum(np.bincount(rows, minlength=A.shape[0]))]).astype(np.int32)
    return off, cols.astype(np.int32), A[rows, cols]


# A(1, 1) cancels exactly in ILU(0): 2 - (4 / 2) * 1 = 0
ILU_ZERO = [[2, 1, 0], [4, 2, 1], [0, 1, 3]]
# IC(0) of the lower triangle: l_11^2 argument 1 - 1 = 0, and 1 - 4 = -3
IC_ZERO = [[1, 1, 0], [1, 1, 0], [0, 0, 2]]
IC_NEG = [[1, 2, 0], [2, 1, 0], [0, 0, 2]]


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
def test_native_zero_pivots(L, dtype):
    off, col, val = small(ILU_ZERO)
    val = val.astype(NP[dtype])
    outs, _, _, pos = native(L, "lu", off, col, val, 0)
    assert pos == 1 == R.factor("lu", off, col, val)[1]
    for on_device in (False, True):
        outs, _, _, pos = native(L, "lu", off, col, val, 0, boost=(1e-8, 0.5), on_device=on_device)
        want, wpos = R.factor("lu", off, col, val, boost=True, tol=1e-8, boost_val=0.5)
        assert pos == wpos == -1 and np.array_equal(outs[0], want)
    for dense in (IC_ZERO, IC_NEG):
        off, col, val = small(dense)
        outs, _, _, pos = native(L, "ic", off, col, val.astype(NP[dtype]), 0)
        assert pos == 1 == R.factor("ic", off, col, val.astype(NP[dtype]))[1]


def test_native_analysis_rejects_bad_patterns(L):
    ws = torch.empty(L.b200ilu0_workspace_bytes(3, 4), dtype=torch.uint8, device="cuda")
    # unsorted, duplicate, out-of-range columns; then offsets past nnz, negative and decreasing (clamped before any kernel reads col)
    for off, col in (([0, 1, 3, 4], [0, 1, 0, 2]), ([0, 1, 3, 4], [0, 1, 1, 2]), ([0, 1, 3, 4], [0, 0, 5, 2]),
                     ([0, 1, 3, 1 << 20], [0, 0, 1, 2]), ([-(1 << 20), 1, 3, 4], [0, 0, 1, 2]), ([0, 3, 1, 4], [0, 0, 1, 2])):
        o, c = torch.tensor(off, dtype=torch.int32, device="cuda"), torch.tensor(col, dtype=torch.int32, device="cuda")
        assert L.b200ilu0_analysis(stream(), 3, 4, o.data_ptr(), c.data_ptr(), 0, ws.data_ptr(), None, None) == -2
    o, c = torch.tensor([0, 1, 2, 3], dtype=torch.int32, device="cuda"), torch.tensor([0, 0, 2], dtype=torch.int32, device="cuda")
    sz = C.c_int64(-9)
    assert L.b200ilu0_analysis(stream(), 3, 3, o.data_ptr(), c.data_ptr(), 0, ws.data_ptr(), C.byref(sz), None) == 0
    assert sz.value == 1


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
@pytest.mark.parametrize("kind", ["lu", "ic"])
def test_native_factor_after_a_structural_zero(L, kind, dtype):
    """Rows without a stored diagonal are left as stored and nothing is read from them: the factor after such an analysis is the
    restatement's bit for bit, canaries hold, and the zero-pivot row is the first structural zero."""
    off, col, val = O.gen_stencil5(100)
    rowof = np.repeat(np.arange(off.size - 1), np.diff(off))
    keep = ~(((rowof == 37) | (rowof == 5000) | (rowof == 9999)) & (col == rowof))
    off = np.concatenate([[0], np.cumsum(np.bincount(rowof[keep], minlength=off.size - 1))]).astype(np.int32)
    col, val = np.asarray(col[keep], np.int32), val[keep].astype(NP[dtype])
    for base in (0, 1):
        outs, sz, lev, pos = native(L, kind, off, col, val, base, runs=2)
        want, wpos = R.factor(kind, off + base, col + base, val, base)
        assert sz == 37 and pos == wpos == 37
        assert np.array_equal(outs[0].view(np.uint8), want.view(np.uint8)) and np.array_equal(outs[1].view(np.uint8), want.view(np.uint8))
    # no entries at all: every row is a structural zero, and the factorization reads no value (values may be NULL)
    off0 = torch.zeros(5, dtype=torch.int32, device="cuda")
    ws = torch.full((L.b200ilu0_workspace_bytes(4, 0) + PAD,), CANARY, dtype=torch.uint8, device="cuda")
    sz, pos = C.c_int64(-9), C.c_int(-7)
    assert L.b200ilu0_analysis(stream(), 4, 0, off0.data_ptr(), None, 0, ws.data_ptr(), C.byref(sz), None) == 0 and sz.value == 0
    assert L.b200ilu0_factor(stream(), KIND[kind], DT[dtype], 4, 0, off0.data_ptr(), None, 0, None, 0, None, None, 0, ws.data_ptr()) == 0
    assert L.b200ilu0_zero_pivot(stream(), ws.data_ptr(), C.byref(pos), 0, None) == 0 and pos.value == 0
    assert (ws[-PAD:] == CANARY).all()


# ---------------------------------------------------------------------------------------------------- through the shim
@pytest.fixture()
def apis(cs):
    ours, closed = cs.Api("b200"), cs.Api("cusparse")
    ours.set_option("B200SPMV_ILU0", "on")
    yield ours, closed
    ours.set_option("B200SPMV_ILU0", "auto")


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
@pytest.mark.parametrize("kind", ["csric02", "csrilu02"])
def test_shim_native_agrees_with_the_closed_library(cs, apis, kind, dtype):
    ours, closed = apis
    if kind == "csric02":
        off, col, val = O.gen_stencil5(700)
    else:
        off, col, val = O.gen_stencil5(700, mass=0.3, ux=0.3, uy=0.2)
    m = off.size - 1
    offd, cold = torch.tensor(off, device="cuda"), torch.tensor(col, device="cuda")
    res = []
    for api in (ours, closed):
        v = torch.tensor(val, dtype=dtype, device="cuda")
        api.reset_stats() if api is ours else None
        out = getattr(cs, kind)(api, m, offd, cold, v)
        res.append((v.double().cpu().numpy(), out))
    st = ours.stats()
    assert st["native"] == 1 and st["forwarded"] == 0 and st["analyze"] == 1, st
    (a, oa), (b, ob) = res
    assert oa["structural"] == ob["structural"] == (0, -1) and oa["numerical"] == ob["numerical"] == (0, -1)
    rel = np.linalg.norm(a - b) / np.linalg.norm(b)
    assert rel < (1e-12 if dtype == torch.float64 else 1e-5), rel
    want, _ = R.factor("ic" if kind == "csric02" else "lu", off, col, val.astype(NP[dtype]))
    assert np.array_equal(a.astype(NP[dtype]), want)


def statuses(cs, api, kind, dense, dtype, pointer_mode, boost=None, missing_diag=False):
    off, col, val = small(dense)
    if missing_diag:                                      # row 2 without its diagonal
        keep = ~((np.repeat(np.arange(3), np.diff(off)) == 2) & (col == 2))
        rowof = np.repeat(np.arange(3), np.diff(off))[keep]
        col, val = col[keep], val[keep]
        off = np.concatenate([[0], np.cumsum(np.bincount(rowof, minlength=3))]).astype(np.int32)
    v = torch.tensor(val, dtype=dtype, device="cuda")
    kw = dict(pointer_mode=pointer_mode)
    if boost is not None:
        kw["boost"] = boost
    out = getattr(cs, kind)(api, 3, torch.tensor(off, device="cuda"), torch.tensor(col, device="cuda"), v, **kw)
    return out["structural"], out["numerical"]


@pytest.mark.parametrize("pointer_mode", [0, 1])
@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
def test_zero_pivot_statuses_are_the_closed_librarys(cs, apis, dtype, pointer_mode):
    ours, closed = apis
    for kind, dense, boost in (("csrilu02", ILU_ZERO, None), ("csrilu02", ILU_ZERO, (1e-8, 0.5)), ("csric02", IC_ZERO, None),
                               ("csric02", IC_NEG, None)):
        a = statuses(cs, ours, kind, dense, dtype, pointer_mode, boost)
        b = statuses(cs, closed, kind, dense, dtype, pointer_mode, boost)
        print(kind, dense, boost, pointer_mode, "closed:", b, "ours:", a)
        assert a == b, (kind, dense, boost, a, b)
    # a missing diagonal is forwarded: the closed library's structural-zero verdict stands
    ours.reset_stats()
    a = statuses(cs, ours, "csrilu02", ILU_ZERO, dtype, pointer_mode, missing_diag=True)
    b = statuses(cs, closed, "csrilu02", ILU_ZERO, dtype, pointer_mode, missing_diag=True)
    assert a == b and ours.stats()["native"] == 0, (a, b)


@pytest.mark.parametrize("kind", ["csric02", "csrilu02"])
def test_default_mode_does_no_native_work(cs, kind):
    """With the default routing no class is native, so bufferSize returns the closed library's size and analysis runs no native
    analysis: the shim only counts and forwards."""
    off, col, val = O.gen_stencil5(200)
    offd, cold = torch.tensor(off, device="cuda"), torch.tensor(col, device="cuda")
    ours, closed = cs.Api("b200"), cs.Api("cusparse")
    ours.set_option("B200SPMV_ILU0", "auto")
    ours.reset_stats()
    vo, vc = torch.tensor(val, device="cuda"), torch.tensor(val, device="cuda")
    a = getattr(cs, kind)(ours, off.size - 1, offd, cold, vo)
    b = getattr(cs, kind)(closed, off.size - 1, offd, cold, vc)
    assert ours.stats() == dict(native=0, forwarded=2, analyze=0), ours.stats()
    assert a == b and a["buffer_size"] == b["buffer_size"], (a, b)
    assert torch.equal(vo, vc)


def test_null_buffer_is_refused(cs, apis):
    # The closed analysis is not run with a NULL buffer: it may write through it.  Ours refuses the call before any CUDA work.
    ours, _ = apis
    off, col, val = small(ILU_ZERO)
    with pytest.raises(cs.CuSparseError) as e:
        cs.csrilu02(ours, 3, torch.tensor(off, device="cuda"), torch.tensor(col, device="cuda"),
                    torch.tensor(val, device="cuda"), buffer=None)
    assert e.value.status == cs.CUSPARSE_STATUS_INVALID_VALUE


# ---------------------------------------------------------------------------------------------------- samples
def clean_env(**extra):
    env = {k: v for k, v in os.environ.items() if k != "B200SPMV_CUSPARSE"}
    env.update(extra)
    return env


@pytest.mark.parametrize("name,iters,what", [("cg", 39, "csric02"), ("bicgstab", 13, "csrilu02")])
def test_solver_samples_factorize_natively(name, iters, what):
    exe = os.path.join(ROOT, "oracle", "_ref", f"{name}_example.b200spsv")
    if not os.path.exists(exe):
        pytest.skip("oracle/_ref not built")
    golden = json.load(open(os.path.join(ROOT, "tests", "golden", "solver_samples.json")))[name]
    p = subprocess.run([exe], capture_output=True, text=True, timeout=300, env=clean_env(B200SPMV_LOG="1", B200SPMV_ILU0="on"))
    assert p.returncode == 0, p.stdout[-2000:] + p.stderr[-2000:]
    lines = [l for l in p.stderr.splitlines() if what in l]
    assert any("analysis native" in l for l in lines) and any(f"D{what} native" in l for l in lines), lines
    assert not any("forwarded" in l for l in lines), lines
    trace = [l for l in p.stdout.splitlines() if "rror" in l or "teration" in l]
    n = sum("teration =" in l or "=== ITERATION" in l.upper() for l in trace)
    assert n == golden["iterations"] == iters, (n, trace[-3:])
    fa = [l for l in p.stdout.splitlines() if "Final error norm" in l]
    va, vb = float(fa[0].split("=")[-1]), golden["final_error_norm"]
    assert abs(va - vb) <= 0.1 * abs(vb) + 1e-12, (fa, vb)
