"""CPU: the numpy restatement of the SpSV plan and its exact fixtures, the routing table of b200spsv_route, the ABI of
libb200spsv.so, and which library each SpSV / SpMV symbol binds to in the opt-in sample binaries."""
import ctypes
import itertools
import os
import subprocess

import numpy as np
import pytest

from oracle import spsv_ref as R
from test_abi import declared_symbols, exported

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "b200spsv.h")
AXES = list(itertools.product((True, False), (False, True), (False, True)))      # lower, unit, transpose


def fixtures():
    """(name, rows, off, col): every matrix shape the GPU tests solve, small enough for the sequential numpy solve."""
    out = [("toy", 4, R.TOY_SPSV["off"], R.TOY_SPSV["col"])]
    for name, (off, col) in (("diagonal", R.diagonal_pattern(37)), ("chain", R.chain_pattern(300)),
                             ("stencil5_9", R.stencil5_pattern(9))):
        out.append((name, off.size - 1, off, col))
    out.append(("n1", 1, np.array([0, 1], np.int32), np.array([0], np.int32)))
    out.append(("n0", 0, np.array([0], np.int32), np.zeros(0, np.int32)))
    out.append(("one_sided",) + ONE_SIDED)
    return out


# Rows 0 and 1 store only their diagonal; row 2 (row 3) stores besides it only an entry of the upper (lower) triangle;
# row 4 stores a single lower entry and no diagonal (UNIT only: with NON_UNIT the analysis hands it to the closed library).
ONE_SIDED = (5, np.array([0, 1, 2, 4, 6, 7], np.int32), np.array([0, 1, 2, 3, 0, 3, 0], np.int32))


@pytest.fixture(scope="module")
def spsv_lib(built_lib):
    from cudalibrarysamples_b200 import build
    lib = ctypes.CDLL(build.SPSV_LIB_PATH)
    lib.b200spsv_csr_workspace_bytes.restype = ctypes.c_size_t
    return lib


# ---------------------------------------------------------------------------------------------------- oracle
def test_reference_toy_golden_comes_out_of_the_numpy_solve():
    T = R.TOY_SPSV
    y = R.solve(T["rows"], T["off"], T["col"], T["val"], T["x"], 1.0, lower=True, unit=False)
    assert np.array_equal(y, T["y_result"])       # spsv_csr_example.c: hY_result = {1, 2, 3, 4}


@pytest.mark.parametrize("lower,unit,transpose", AXES)
@pytest.mark.parametrize("base", [0, 1])
def test_plan_invariants(lower, unit, transpose, base):
    for name, rows, off, col in fixtures():
        p = R.plan(rows, off + base, col + base, base, lower, unit, transpose)
        R.check_plan(rows, off + base, col + base, base, lower, unit, transpose, p)


def test_transposed_plan_rows_ascend_in_the_original_row():
    off, col = R.stencil5_pattern(6)
    p = R.plan(36, off, col, 0, lower=True, transpose=True)
    for i in range(36):
        seg = p["t_col"][p["t_off"][i]:p["t_off"][i + 1]]
        assert np.all(np.diff(seg) > 0)


def test_missing_diagonal_is_counted_for_non_unit_only():
    off, col = np.array([0, 1, 2, 3], np.int32), np.array([0, 0, 2], np.int32)      # row 1 stores no diagonal
    assert R.plan(3, off, col, unit=False)["missing"] == 1
    assert R.plan(3, off, col, unit=True)["missing"] == 0


@pytest.mark.parametrize("kind", ["f32", "f64", "wide"])
@pytest.mark.parametrize("lower,unit,transpose", AXES)
def test_exact_fixtures_solve_to_y_star(kind, lower, unit, transpose):
    for name, rows, off, col in fixtures():
        if name == "one_sided" and not unit:
            continue
        for base in (0, 1):
            val, x, ys, alpha = R.exact_case(rows, off + base, col + base, base, lower, unit, transpose, kind, seed=rows)
            y = R.solve(rows, off + base, col + base, val, x, alpha, base, lower, unit, transpose)
            assert np.array_equal(y, ys), (name, base)


def test_wide_fixture_needs_more_than_fp32():
    off, col = R.chain_pattern(64)
    val, x, ys, alpha = R.exact_case(64, off, col, 0, True, False, False, "wide", seed=1)
    y32 = R.solve(64, off, col, val.astype(np.float32), x.astype(np.float32), alpha, 0, True, False, False)
    assert not np.array_equal(y32.astype(np.float64), ys)


# ---------------------------------------------------------------------------------------------------- routing
CSR, COO, SELL = 1, 4, 6                 # cusparseFormat_t
I32, I64 = 2, 3
F32, F64, F16, C32 = 0, 1, 2, 4          # cudaDataType


def route(lib, fmt=CSR, op=0, alg=0, off=I32, col=I32, a=F64, x=None, y=None, ct=None, fill=0, diag=0, rows=100, cols=None, nnz=500):
    x = a if x is None else x
    y = a if y is None else y
    ct = a if ct is None else ct
    cols = rows if cols is None else cols
    return lib.b200spsv_route(fmt, op, alg, off, col, a, x, y, ct, fill, diag, ctypes.c_int64(rows), ctypes.c_int64(cols),
                              ctypes.c_int64(nnz))


def test_route_table(spsv_lib):
    L = spsv_lib
    for a, op, fill, diag in itertools.product((F32, F64), (0, 1), (0, 1), (0, 1)):
        assert route(L, a=a, op=op, fill=fill, diag=diag) == 1
    assert route(L, rows=0, nnz=0) == 1 and route(L, rows=1, nnz=1) == 1
    assert route(L, fmt=COO) == 0 and route(L, fmt=SELL) == 0
    assert route(L, off=I64) == 0 and route(L, col=I64) == 0 and route(L, off=I64, col=I64) == 0
    assert route(L, a=C32) == 0 and route(L, a=F16) == 0
    assert route(L, a=F32, x=F64, y=F64, ct=F64) == 0 and route(L, a=F64, ct=F32) == 0 and route(L, y=F32) == 0
    assert route(L, op=2) == 0                       # conjugate transpose
    assert route(L, alg=1) == 0
    assert route(L, fill=2) == 0 and route(L, diag=2) == 0
    assert route(L, cols=101) == 0                   # non-square: the closed library's verdict
    assert route(L, rows=2 ** 31, nnz=5) == 0 and route(L, nnz=2 ** 31) == 0


# ---------------------------------------------------------------------------------------------------- ABI
def test_header_declares_the_spsv_entry_points():
    names = declared_symbols(HEADER, "B200SPSV_EXPORT")
    for n in ["cusparseSpSV_createDescr", "cusparseSpSV_destroyDescr", "cusparseSpSV_bufferSize", "cusparseSpSV_analysis",
              "cusparseSpSV_solve", "cusparseSpSV_updateMatrix", "b200spsv_csr_workspace_bytes", "b200spsv_csr_analysis",
              "b200spsv_csr_solve", "b200spsv_csr_params", "b200spsv_csr_layout", "b200spsv_route", "b200spsv_get_stats",
              "b200spsv_reset_stats"]:
        assert n in names, n


def test_spsv_library_exports_every_declared_symbol(spsv_lib):
    from cudalibrarysamples_b200 import build
    have = exported(build.SPSV_LIB_PATH)
    assert not [n for n in declared_symbols(HEADER, "B200SPSV_EXPORT") if n not in have]
    # only SpSV from the cuSPARSE namespace: SpMV and the descriptors keep binding where they did
    assert sorted(n for n in have if n.startswith("cusparse")) == sorted(
        "cusparseSpSV_" + s for s in ("createDescr", "destroyDescr", "bufferSize", "analysis", "solve", "updateMatrix"))


def test_spmv_library_exports_no_spsv(built_lib):
    assert not [n for n in exported(built_lib) if n.startswith("cusparseSpSV") or n.startswith("b200spsv")]


def test_spsv_library_does_not_need_the_spmv_library(spsv_lib):
    from cudalibrarysamples_b200 import build
    out = subprocess.check_output(["readelf", "-d", build.SPSV_LIB_PATH], text=True)
    assert "libb200spmv" not in out and "libcusparse" not in out


def test_host_side_argument_checks(spsv_lib):
    L = spsv_lib
    i64 = ctypes.c_int64
    ws = ctypes.c_void_p(1 << 20)                                   # never dereferenced: every call below fails first
    assert L.b200spsv_csr_analysis(None, i64(-1), i64(0), None, None, 0, 1, 0, 0, ws, None) == -1
    assert L.b200spsv_csr_analysis(None, i64(4), i64(9), None, None, 0, 1, 0, 0, ws, None) == -1      # no arrays
    assert L.b200spsv_csr_analysis(None, i64(4), i64(9), ws, ws, 2, 1, 0, 0, ws, None) == -1          # base 2
    assert L.b200spsv_csr_analysis(None, i64(4), i64(9), ws, ws, 0, 1, 0, 0, None, None) == -1        # no workspace
    assert L.b200spsv_csr_analysis(None, i64(4), i64(9), ws, ws, 0, 1, 0, 0, ctypes.c_void_p((1 << 20) + 4), None) == -1
    one = ctypes.c_double(1.0)
    assert L.b200spsv_csr_solve(None, 7, i64(4), i64(9), 1, 0, 0, ws, None, ctypes.byref(one), 0, ws, ws, ws) == -1   # dtype
    assert L.b200spsv_csr_solve(None, 1, i64(4), i64(9), 1, 0, 0, ws, None, None, 0, ws, ws, ws) == -1              # alpha
    assert L.b200spsv_csr_solve(None, 1, i64(4), i64(9), 1, 0, 0, ws, None, ctypes.byref(one), 0, None, ws, ws) == -1
    assert L.b200spsv_csr_solve(None, 1, i64(4), i64(9), 3, 0, 0, ws, None, ctypes.byref(one), 0, ws, ws, ws) == -1 # lower
    assert L.b200spsv_csr_solve(None, 1, i64(0), i64(0), 1, 0, 0, None, None, None, 0, None, None, ws) == 0         # empty
    off = (ctypes.c_size_t * 8)()
    assert L.b200spsv_csr_layout(i64(-1), i64(0), 0, off) == -1


def test_layout_and_params(spsv_lib):
    L = spsv_lib
    for rows, nnz, tr in ((0, 0, 0), (1, 1, 1), (1000, 4978, 0), (1000, 4978, 1), (64, 64, 0)):
        off = (ctypes.c_size_t * 8)()
        assert L.b200spsv_csr_layout(ctypes.c_int64(rows), ctypes.c_int64(nnz), tr, off) == 0
        o = list(off)
        assert o[0] == 0 and all(v % 256 == 0 for v in o) and o == sorted(o)
        assert o[1] - o[0] >= 16 and o[2] - o[1] >= 4 * rows and o[3] - o[2] >= 4 * (rows + 1)
        assert o[4] - o[3] >= 4 * rows and o[5] - o[4] >= 4 * nnz and o[6] - o[5] >= 4 * nnz
        assert o[7] - o[6] >= 4 * rows + (8 * nnz if tr else 0)
        assert L.b200spsv_csr_workspace_bytes(ctypes.c_int64(rows), ctypes.c_int64(nnz), tr) == o[7]
    t, b = ctypes.c_int32(), ctypes.c_uint64()
    L.b200spsv_csr_params(ctypes.byref(t), ctypes.byref(b))
    assert t.value % 32 == 0 and t.value > 0 and 10 ** 9 <= b.value <= 60 * 10 ** 9


# ---------------------------------------------------------------------------------------------------- bindings
def _bindings(exe, **env):
    e = {k: v for k, v in os.environ.items() if k != "B200SPMV_CUSPARSE"}
    e.update(LD_BIND_NOW="1", LD_DEBUG="bindings", **env)
    p = subprocess.run([exe], env=e, capture_output=True, text=True, timeout=120)
    name = os.path.basename(exe)
    lines = [l for l in p.stderr.splitlines() if f"{name} [0] to" in l]

    def target(sym):
        return [l for l in lines if f"`{sym}'" in l][0]
    return target


def test_opt_in_sample_binds_spsv_to_the_spsv_library():
    exe = os.path.join(ROOT, "oracle", "_ref", "cg_example.b200spsv")
    if not os.path.exists(exe):
        pytest.skip("oracle/_ref not built (needs the reference checkout)")
    target = _bindings(exe)
    for s in ("cusparseSpSV_solve", "cusparseSpSV_analysis", "cusparseSpSV_bufferSize", "cusparseSpSV_createDescr"):
        assert "libb200spsv.so" in target(s), s
    assert "libb200spmv.so" in target("cusparseSpMV")
    assert "libb200spmv.so" in target("cusparseCreateCsr")
    assert "libcusparse.so.12" in target("cusparseCreate")
    assert "libcusparse.so.12" in target("cusparseSpMatSetAttribute")


def test_preloading_the_spsv_library_moves_only_spsv():
    exe = os.path.join(ROOT, "oracle", "_ref", "cg_example.cusparse")
    lib = os.path.join(ROOT, "cudalibrarysamples_b200", "libb200spsv.so")
    if not (os.path.exists(exe) and os.path.exists(lib)):
        pytest.skip("oracle/_ref or the library not built")
    target = _bindings(exe, LD_PRELOAD=lib)
    assert "libb200spsv.so" in target("cusparseSpSV_solve")
    assert "libcusparse.so.12" in target("cusparseSpMV")
    assert "libcusparse.so.12" in target("cusparseCreateCsr")
