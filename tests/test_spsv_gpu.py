"""GPU: the native CSR triangular solve of libb200spsv.so (cusparseSpSV_*) against exact fixtures bit for bit, against the
numpy plan bit for bit, and against the closed library on inexact data; repeatability and graph replay; forwarded cases;
the opt-in sample binaries.  Every native solve must leave the error word at 0 and forward nothing."""
import ctypes as C
import itertools
import json
import os
import subprocess

import numpy as np
import pytest
import torch

from cudalibrarysamples_b200 import cusparse_api as cs
from cudalibrarysamples_b200 import lib as _lib
from oracle import oracle as O
from oracle import spsv_ref as R

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEV = torch.device("cuda:0")
LOWER, UPPER = cs.CUSPARSE_FILL_MODE_LOWER, cs.CUSPARSE_FILL_MODE_UPPER
NON_UNIT, UNIT = cs.CUSPARSE_DIAG_TYPE_NON_UNIT, cs.CUSPARSE_DIAG_TYPE_UNIT
NT, TR = cs.CUSPARSE_OPERATION_NON_TRANSPOSE, cs.CUSPARSE_OPERATION_TRANSPOSE
TD = {np.float32: torch.float32, np.float64: torch.float64}


def t(a):
    return torch.tensor(np.ascontiguousarray(a), device=DEV)


def arrays(off, col, val):
    return dict(off=t(off), col=t(col), val=t(val))


def rmat_reversed(n=8192):
    """R-MAT with its indices reversed (hub rows / columns move to the end) plus the diagonal: its lower triangle has
    rows with more than 32 and more than 1000 dependencies and hub columns."""
    off, col, _ = O.rmat_csr(n, avg_nnz=16, seed=5, val_seed=6)
    r = np.repeat(np.arange(n), np.diff(off))
    return R.coo_to_csr(n, np.concatenate([n - 1 - r, np.arange(n)]), np.concatenate([n - 1 - col, np.arange(n)]))


def matrices():
    out = {"toy": (4, R.TOY_SPSV["off"], R.TOY_SPSV["col"]),
           "diagonal": (1000,) + R.diagonal_pattern(1000),
           "chain": (20000,) + R.chain_pattern(20000),          # > 132 SMs x 64 resident warps of dependency levels
           "stencil64": (64 * 64,) + R.stencil5_pattern(64),
           "n1": (1, np.array([0, 1], np.int32), np.array([0], np.int32)),
           "one_sided": (5, np.array([0, 1, 2, 4, 6, 7], np.int32), np.array([0, 1, 2, 3, 0, 3, 0], np.int32))}
    return out


MATS = matrices()
_BIG = {}


def big(name):
    if name not in _BIG:
        _BIG[name] = (700 * 700,) + R.stencil5_pattern(700) if name == "stencil700" else (8192,) + rmat_reversed()
    return _BIG[name]


def ws_arrays(lib, s, rows, nnz, transpose):
    """The plan and state words in the solver's buffer, read through the layout query."""
    off = (C.c_size_t * 8)()
    assert lib.b200spsv_csr_layout(C.c_int64(rows), C.c_int64(nnz), int(transpose), off) == 0
    buf = s.buffer.cpu().numpy()

    def i32(k, n):
        return buf[off[k]:off[k] + 4 * n].view(np.int32)
    t_off = i32(2, rows + 1)
    tn = int(t_off[-1])
    return dict(state=buf[off[0]:off[0] + 16].view(np.uint32), flags=buf[off[1]:off[1] + 4 * rows].view(np.uint32), t_off=t_off,
                diag_vidx=i32(3, rows), t_col=i32(4, tn), t_vidx=i32(5, tn))


def check_state(lib, s, rows, nnz, transpose, solves):
    w = ws_arrays(lib, s, rows, nnz, transpose)
    st = w["state"]
    assert st[2] == 0, "a wait ran out of its budget"
    assert st[0] == solves and (rows == 0 or st[1] >= rows), st          # epoch == solves so far, every row claimed
    assert np.all(w["flags"] == solves)
    return w


def run_exact(name, rows, off, col, lower, unit, op, kind, base, dev_alpha, check_plan=True):
    api = cs.Api("b200")
    val, x, ys, alpha = R.exact_case(rows, off + base, col + base, base, lower, unit, op == TR, kind, seed=rows + base)
    api.reset_spsv_stats()
    s = cs.SpSVSolver(api, rows, arrays(off + base, col + base, val), fill=LOWER if lower else UPPER,
                      diag=UNIT if unit else NON_UNIT, op=op, base=base, device_alpha=dev_alpha)
    y = torch.full((max(rows, 1),), float("nan"), dtype=TD[val.dtype.type], device=DEV)
    a = torch.tensor([alpha], dtype=y.dtype, device=DEV) if dev_alpha else alpha
    s(t(x) if rows else torch.zeros(1, dtype=y.dtype, device=DEV), y, a)
    torch.cuda.synchronize()
    assert np.array_equal(y.cpu().numpy()[:rows], ys), (name, kind)
    st = api.spsv_stats()
    assert st["forwarded"] == 0 and st["native"] == 1 and st["analysis"] == 1, st
    w = check_state(_lib.spsv(), s, rows, int(off[-1]), op == TR, 1)
    if check_plan:
        p = R.plan(rows, off + base, col + base, base, lower, unit, op == TR)
        for k in ("t_off", "t_col", "t_vidx", "diag_vidx"):
            assert np.array_equal(w[k], p[k]), k
    s.close()


AXES = list(itertools.product((True, False), (False, True), (NT, TR)))


@pytest.mark.parametrize("dev_alpha", [False, True])
@pytest.mark.parametrize("base", [0, 1])
@pytest.mark.parametrize("kind", ["f32", "f64", "wide"])
@pytest.mark.parametrize("lower,unit,op", AXES)
@pytest.mark.parametrize("name", list(MATS))
def test_exact_solve_and_plan(name, lower, unit, op, kind, base, dev_alpha):
    rows, off, col = MATS[name]
    if name == "one_sided" and not unit:
        pytest.skip("row 4 stores no diagonal: NON_UNIT is forwarded (test_forwarded_cases)")
    run_exact(name, rows, off, col, lower, unit, op, kind, base, dev_alpha)


@pytest.mark.parametrize("lower,unit,op", AXES)
@pytest.mark.parametrize("name", ["stencil700", "rmat"])
def test_exact_solve_large(name, lower, unit, op):
    rows, off, col = big(name)
    for kind, base in (("f32", 0), ("wide", 1)):
        run_exact(name, rows, off, col, lower, unit, op, kind, base, False)


def test_n0():
    api = cs.Api("b200")
    api.reset_spsv_stats()
    a = arrays(np.array([0], np.int32), np.zeros(1, np.int32), np.zeros(1))
    a["col"], a["val"] = a["col"][:0], a["val"][:0]
    s = cs.SpSVSolver(api, 0, a)
    y = torch.full((1,), 7.0, dtype=torch.float64, device=DEV)
    s(torch.ones(1, dtype=torch.float64, device=DEV), y, 1.0)
    torch.cuda.synchronize()
    assert y.item() == 7.0 and api.spsv_stats()["forwarded"] == 0
    s.close()


# ---------------------------------------------------------------------------------------------------- vs the closed library
def dominant(off, col, dtype, seed):
    """Values with a dominant diagonal, for either triangle: |d_i| = 1 + sum of |row i| (both triangles)."""
    rows = off.size - 1
    v = O.uniform(seed, int(off[-1]), np.float64)
    r = np.repeat(np.arange(rows), np.diff(off))
    d = col == r
    v[d] = 0
    v[d] = (1.0 + np.bincount(r, weights=np.abs(v), minlength=rows))[r[d]] * np.where(np.arange(d.sum()) % 2, 1, -1)
    return v.astype(dtype)


def pair(rows, a, fill, diag, op, x, alpha=1.0, mat_hook=None):
    """The same solve through our library and the closed one, on the same device buffers."""
    out = []
    for impl in ("b200", "cusparse"):
        api = cs.Api(impl)
        s = cs.SpSVSolver(api, rows, a, fill=fill, diag=diag, op=op)
        if mat_hook:
            mat_hook(api, s)
        y = torch.full_like(x, float("nan"))
        s(x, y, alpha)
        torch.cuda.synchronize()
        out.append(y.cpu().numpy())
        s.close()
    return out


def rel(a, b):
    return np.linalg.norm(a - b) / np.linalg.norm(b)


@pytest.mark.parametrize("dtype,tol", [(np.float64, 1e-12), (np.float32, 1e-5)])
@pytest.mark.parametrize("fill,diag,op", list(itertools.product((LOWER, UPPER), (NON_UNIT, UNIT), (NT, TR))))
def test_matches_closed_library(dtype, tol, fill, diag, op):
    for grid, kw in ((700, {}), (64, dict(mass=0.3, ux=0.3, uy=0.2))):      # cg's matrix, bicgstab's matrix
        off, col, val = O.gen_stencil5(grid, **kw)
        rows = off.size - 1
        v = dominant(off, col, dtype, grid) if diag == NON_UNIT else (val / (np.abs(val).max() * 5)).astype(dtype)
        x = t(O.uniform(grid + 1, rows, dtype))
        api = cs.Api("b200")
        api.reset_spsv_stats()
        ours, ref = pair(rows, arrays(off, col, v), fill, diag, op, x, 0.5)
        assert api.spsv_stats()["forwarded"] == 0
        assert rel(ours, ref) < tol


def test_bicgstab_factors_and_rmat_match_closed_library():
    off, col, val = O.gen_stencil5(128, mass=0.3, ux=0.3, uy=0.2)
    rows = off.size - 1
    v = dominant(off, col, np.float64, 3)
    x = t(O.uniform(4, rows))
    for fill, diag in ((LOWER, UNIT), (UPPER, NON_UNIT)):                    # matM_lower / matM_upper over one pattern
        ours, ref = pair(rows, arrays(off, col, v), fill, diag, NT, x)
        assert rel(ours, ref) < 1e-12
    rows, off, col = big("rmat")
    v = dominant(off, col, np.float64, 9)
    x = t(O.uniform(10, rows))
    for op in (NT, TR):
        ours, ref = pair(rows, arrays(off, col, v), LOWER, NON_UNIT, op, x)
        assert rel(ours, ref) < 1e-12


# ---------------------------------------------------------------------------------------------------- reuse
def test_repeated_solves_and_graph_replay_give_identical_bits():
    off, col, val = O.gen_stencil5(300)
    rows = off.size - 1
    v = dominant(off, col, np.float64, 1)
    api = cs.Api("b200")
    stream = torch.cuda.Stream()
    with torch.cuda.stream(stream):
        s = cs.SpSVSolver(api, rows, arrays(off, col, v), op=TR)
        x = t(O.uniform(2, rows))
        y = torch.empty(rows, dtype=torch.float64, device=DEV)
        s(x, y, 1.0)
        stream.synchronize()
        first = y.cpu().numpy().copy()
        for _ in range(20):
            y.fill_(float("nan"))
            s(x, y, 1.0)
            stream.synchronize()
            assert np.array_equal(y.cpu().numpy(), first)
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=stream):
            s(x, y, 1.0)
        for _ in range(3):
            y.fill_(float("nan"))
            g.replay()
            stream.synchronize()
            assert np.array_equal(y.cpu().numpy(), first)
    check_state(_lib.spsv(), s, rows, off[-1], True, 21 + 3)
    s.close()


def test_two_descriptors_on_one_matrix_as_cg():
    """cg_example.c: L and L^T solves on one matL, separate SpSV descriptors and buffers; z = L^-T L^-1 r."""
    off, col, val = O.gen_stencil5(200)
    rows = off.size - 1
    v = dominant(off, col, np.float64, 5)
    r = t(O.uniform(6, rows))
    res = []
    for impl in ("b200", "cusparse"):
        api = cs.Api(impl)
        h = api.cusparseCreate()
        a = arrays(off, col, v)
        mat = api.cusparseCreateCsr(rows, rows, int(off[-1]), a["off"], a["col"], a["val"])
        api.cusparseSpMatSetAttribute(mat, cs.CUSPARSE_SPMAT_FILL_MODE, LOWER)
        api.cusparseSpMatSetAttribute(mat, cs.CUSPARSE_SPMAT_DIAG_TYPE, NON_UNIT)
        sl = cs.SpSVSolver(api, rows, a, handle=h, mat=mat, op=NT)
        slt = cs.SpSVSolver(api, rows, a, handle=h, mat=mat, op=TR)
        tmp, z = torch.empty_like(r), torch.empty_like(r)
        sl(r, tmp)
        slt(tmp, z)
        torch.cuda.synchronize()
        res.append(z.cpu().numpy())
        sl.close(), slt.close()
        api.cusparseDestroySpMat(mat)
        api.cusparseDestroy(h)
    assert rel(res[0], res[1]) < 1e-12


@pytest.mark.parametrize("change", ["xy", "setvalues", "general", "diagonal", "inplace"])
def test_value_changes_follow_the_closed_library(change):
    """New x / y, new values through cusparseSpMatSetValues or cusparseSpSV_updateMatrix (GENERAL, DIAGONAL), and x == y:
    each must give what the closed library gives after the same call."""
    off, col = R.stencil5_pattern(50)
    rows = off.size - 1
    v0 = dominant(off, col, np.float64, 11)
    v1 = t(dominant(off, col, np.float64, 12))
    dnew = t(2.0 + O.uniform(13, rows))
    x = t(O.uniform(14, rows))
    out = []
    for impl in ("b200", "cusparse"):
        api = cs.Api(impl)
        if impl == "b200":
            api.reset_spsv_stats()
        a = arrays(off, col, v0)
        s = cs.SpSVSolver(api, rows, a)
        if change == "setvalues":
            api.cusparseSpMatSetValues(s.mat, v1)
        elif change == "general":
            s.update(v1, cs.CUSPARSE_SPSV_UPDATE_GENERAL)
        elif change == "diagonal":
            s.update(dnew, cs.CUSPARSE_SPSV_UPDATE_DIAGONAL)
        if change == "inplace":
            y = x.clone()
            s(y, y, 1.0)
        else:
            y = torch.full_like(x, float("nan"))
            s(x, y, 1.0)
        torch.cuda.synchronize()
        out.append(y.cpu().numpy())
        if impl == "b200":
            assert api.spsv_stats()["forwarded"] == 0
            check_state(_lib.spsv(), s, rows, off[-1], False, 1)
        s.close()
    assert rel(out[0], out[1]) < 1e-12, change


def test_stored_zero_diagonal_gives_the_closed_librarys_non_finite_mask():
    off, col = R.chain_pattern(64)
    v = dominant(off, col, np.float64, 21)
    r = np.repeat(np.arange(64), np.diff(off))
    v[(col == r) & (r == 20)] = 0.0
    x = t(O.uniform(22, 64))
    ours, ref = pair(64, arrays(off, col, v), LOWER, NON_UNIT, NT, x)
    assert np.array_equal(np.isnan(ours), np.isnan(ref)) and np.array_equal(np.isinf(ours), np.isinf(ref))
    ok = np.isfinite(ref)
    assert np.allclose(ours[ok], ref[ok], rtol=1e-12, atol=0)


# ---------------------------------------------------------------------------------------------------- forwarded
def generic_solve(api, mat, rows, x, dtype=torch.float64):
    h = api.cusparseCreate()
    api.cusparseSpMatSetAttribute(mat, cs.CUSPARSE_SPMAT_FILL_MODE, LOWER)
    api.cusparseSpMatSetAttribute(mat, cs.CUSPARSE_SPMAT_DIAG_TYPE, NON_UNIT)
    y = torch.zeros(rows, dtype=dtype, device=DEV)
    vx, vy = api.cusparseCreateDnVec(rows, x), api.cusparseCreateDnVec(rows, y)
    d = api.cusparseSpSV_createDescr()
    ct = cs._VT[dtype]
    size = api.cusparseSpSV_bufferSize(h, NT, 1.0, mat, vx, vy, ct, 0, d)
    buf = torch.empty(max(size, 16), dtype=torch.uint8, device=DEV)
    api.cusparseSpSV_analysis(h, NT, 1.0, mat, vx, vy, ct, 0, d, buf)
    api.cusparseSpSV_solve(h, NT, 1.0, mat, vx, vy, ct, 0, d)
    torch.cuda.synchronize()
    api.cusparseSpSV_destroyDescr(d)
    api.cusparseDestroyDnVec(vx), api.cusparseDestroyDnVec(vy)
    api.cusparseDestroy(h)
    return y.cpu().numpy()


@pytest.mark.parametrize("case", ["coo", "sell", "idx64", "missing_diag"])
def test_forwarded_cases(case):
    T = O.TOY
    res = []
    for impl in ("b200", "cusparse"):
        api = cs.Api(impl)
        x = t(R.TOY_SPSV["x"].astype(np.float32))
        if case == "coo":
            mat = api.cusparseCreateCoo(4, 4, 9, t(T["coo_row"]), t(T["csr_col"]), t(T["val"]))
        elif case == "sell":
            mat = api.cusparseCreateSlicedEll(4, 4, 9, 12, 2, t(T["sell_off"]), t(T["sell_col"]), t(T["sell_val"]))
        elif case == "idx64":
            mat = api.cusparseCreateCsr(4, 4, 9, t(T["csr_off"].astype(np.int64)), t(T["csr_col"].astype(np.int64)), t(T["val"]))
        else:                                  # row 1 stores no diagonal: ((0,0),(1,0),(2,2)) -> LOWER NON_UNIT is ill-posed
            off, col = np.array([0, 1, 2, 3], np.int32), np.array([0, 0, 2], np.int32)
            mat = api.cusparseCreateCsr(3, 3, 3, t(off), t(col), t(np.array([2, 1, 4], np.float32)))
            x = x[:3].contiguous()
        if impl == "b200":
            api.reset_spsv_stats()
        y = generic_solve(api, mat, x.numel(), x, torch.float32)
        if impl == "b200":
            st = api.spsv_stats()
            assert st["forwarded"] > 0 and st["native"] == 0, st
        api.cusparseDestroySpMat(mat)
        res.append(y)
    assert np.array_equal(np.isnan(res[0]), np.isnan(res[1]))
    ok = np.isfinite(res[1])
    assert np.array_equal(res[0][ok], res[1][ok]), (case, res)


def statuses(fn):
    out = []
    for impl in ("b200", "cusparse"):
        try:
            fn(cs.Api(impl))
            out.append(0)
        except cs.CuSparseError as e:
            out.append(e.status)
    return out


def test_statuses_follow_the_closed_library():
    def non_square(api):
        h = api.cusparseCreate()
        a = arrays(np.array([0, 1, 2], np.int32), np.array([0, 1], np.int32), np.ones(2))
        mat = api.cusparseCreateCsr(2, 3, 2, a["off"], a["col"], a["val"])
        try:
            x, y = torch.ones(3, dtype=torch.float64, device=DEV), torch.ones(2, dtype=torch.float64, device=DEV)
            vx, vy = api.cusparseCreateDnVec(3, x), api.cusparseCreateDnVec(2, y)
            d = api.cusparseSpSV_createDescr()
            api.cusparseSpSV_bufferSize(h, NT, 1.0, mat, vx, vy, cs.CUDA_R_64F, 0, d)
        finally:
            api.cusparseDestroySpMat(mat)

    def null_buffer(api):
        h = api.cusparseCreate()
        off, col = R.chain_pattern(8)
        a = arrays(off, col, dominant(off, col, np.float64, 1))
        mat = api.cusparseCreateCsr(8, 8, int(off[-1]), a["off"], a["col"], a["val"])
        api.cusparseSpMatSetAttribute(mat, cs.CUSPARSE_SPMAT_FILL_MODE, LOWER)
        x, y = torch.ones(8, dtype=torch.float64, device=DEV), torch.ones(8, dtype=torch.float64, device=DEV)
        vx, vy = api.cusparseCreateDnVec(8, x), api.cusparseCreateDnVec(8, y)
        d = api.cusparseSpSV_createDescr()
        try:
            api.cusparseSpSV_analysis(h, NT, 1.0, mat, vx, vy, cs.CUDA_R_64F, 0, d, None)
        finally:
            api.cusparseDestroySpMat(mat)

    a, b = statuses(non_square)
    assert a == b and b != 0
    # A NULL buffer at analysis: the closed library accepts it and its analysis kernels then write through it, so it is
    # not run here; ours refuses the call before any CUDA work.
    with pytest.raises(cs.CuSparseError) as e:
        null_buffer(cs.Api("b200"))
    assert e.value.status == cs.CUSPARSE_STATUS_INVALID_VALUE


# ---------------------------------------------------------------------------------------------------- samples
def clean_env(**extra):
    env = {k: v for k, v in os.environ.items() if k != "B200SPMV_CUSPARSE"}
    env.update(extra)
    return env


def test_spsv_sample_runs_natively():
    exe = os.path.join(ROOT, "oracle", "_ref", "spsv_csr_example.b200spsv")
    if not os.path.exists(exe):
        pytest.skip("oracle/_ref not built")
    p = subprocess.run([exe], capture_output=True, text=True, timeout=120, env=clean_env(B200SPMV_LOG="1"))
    assert p.returncode == 0, p.stdout + p.stderr
    assert "spsv_csr_example test PASSED" in p.stdout
    assert "[b200spsv] solve native" in p.stderr and "forwarded" not in p.stderr


@pytest.mark.parametrize("name,iters", [("cg", 39), ("bicgstab", 13)])
def test_solver_samples_with_native_spsv_reproduce_the_trace(name, iters):
    exe = os.path.join(ROOT, "oracle", "_ref", f"{name}_example.b200spsv")
    if not os.path.exists(exe):
        pytest.skip("oracle/_ref not built")
    golden = json.load(open(os.path.join(ROOT, "tests", "golden", "solver_samples.json")))[name]
    p = subprocess.run([exe], capture_output=True, text=True, timeout=300, env=clean_env(B200SPMV_LOG="1"))
    assert p.returncode == 0, p.stdout[-2000:] + p.stderr[-2000:]
    spsv_lines = [l for l in p.stderr.splitlines() if l.startswith("[b200spsv]")]
    assert any("solve native" in l for l in spsv_lines) and not any("forwarded" in l for l in spsv_lines)
    trace = [l for l in p.stdout.splitlines() if "rror" in l or "teration" in l]
    n = sum("teration =" in l or "=== ITERATION" in l.upper() for l in trace)
    assert n == golden["iterations"] == iters, (n, trace[-3:])
    fa = [l for l in p.stdout.splitlines() if "Final error norm" in l]
    va, vb = float(fa[0].split("=")[-1]), golden["final_error_norm"]
    assert abs(va - vb) <= 0.1 * abs(vb) + 1e-12, (fa, vb)
