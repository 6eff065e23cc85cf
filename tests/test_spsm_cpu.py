"""CPU: the numpy restatement of cusparseSpSM (oracle/spsm_ref.py) against scipy, the level order on hand-checked patterns, the
routing table of b200spsm_route, the layout and argument checks of the b200spsm_* entry points, the exports of libb200spmv.so, and
which library the opt-in spsm_csr sample binds to."""
import ctypes
import itertools
import os

import numpy as np
import pytest
import scipy.sparse as sp
import scipy.sparse.linalg as sl

from oracle import spsm_ref as M
from test_abi import declared_symbols, exported

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
AXES = list(itertools.product((True, False), (False, True), (False, True)))      # lower, unit, transpose


@pytest.fixture(scope="module")
def L(built_lib):
    from cudalibrarysamples_b200 import lib
    return lib.shim()


def triangle(rows, off, col, val, lower, unit, transpose):
    """The dense op(T) scipy solves with."""
    A = sp.csr_matrix((val.astype(np.float64), col, off), shape=(rows, rows)).toarray()
    T = np.tril(A, -1) if lower else np.triu(A, 1)
    T = T + (np.eye(rows) if unit else np.diag(np.diag(A)))
    return T.T if transpose else T


# ---------------------------------------------------------------------------------------------------- oracle
def test_toy_golden_comes_out_of_the_restatement():
    T = M.TOY_SPSM
    for w in (1, 2, 8, 32):
        C = M.solve(4, T["off"], T["col"], T["val"], T["B"].reshape(2, 4).T, 1.0, w=w)
        assert np.array_equal(C.T.ravel(), T["C_result"])      # spsm_csr_example.c: hY_result = {1, 2, 3, 4} twice


@pytest.mark.parametrize("lower,unit,transpose", AXES)
@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_restatement_matches_scipy(lower, unit, transpose, dtype):
    rng = np.random.default_rng(3)
    for name, rows, off, col in M.fixtures():
        val = M.values(rows, off, col, dtype, seed=rows)
        T = triangle(rows, off, col, val, lower, unit, transpose)
        for nrhs, w in ((1, 1), (3, 4), (33, 32), (5, 8)):
            B = rng.uniform(-1, 1, (rows, nrhs)).astype(dtype)
            for base in (0, 1):
                C = M.solve(rows, off + base, col + base, val, B, 0.5, base, lower, unit, transpose, w)
                want = sl.spsolve_triangular(sp.csr_matrix(T), 0.5 * B.astype(np.float64), lower=lower != transpose,
                                             unit_diagonal=False)
                tol = 1e-4 if dtype == np.float32 else 1e-12
                assert np.allclose(C, want, rtol=tol, atol=tol), (name, nrhs, base)


def test_tile_width_changes_only_the_grouping():
    off, col = M.SR.stencil5_pattern(9)
    val = M.values(81, off, col, np.float64, seed=1)
    B = np.random.default_rng(0).uniform(-1, 1, (81, 40))
    ref = M.solve(81, off, col, val, B, 1.0, w=1)
    for w in (2, 4, 8, 16, 32):
        assert np.allclose(M.solve(81, off, col, val, B, 1.0, w=w), ref, rtol=1e-13, atol=1e-13)


def test_long_rows_fixture_makes_the_summation_order_visible():
    """On the long-row fixture every tile width gives different bits (the restatement is sensitive to the grouping), each group
    sums several entries at every width, and a contiguous split of the entries instead of the strided one changes the bits too."""
    rows, off, col = [(r, o, c) for n, r, o, c in M.fixtures() if n == "long_rows"][0]
    for lower, tr in ((True, False), (False, False), (True, True), (False, True)):
        p = M.plan(rows, off, col, 0, lower, False, tr)
        assert np.diff(p["t_off"]).max() > 64
    val = M.values(rows, off, col, np.float32, seed=1)
    B = np.random.default_rng(2).uniform(-1, 1, (rows, 3)).astype(np.float32)
    out = {w: M.solve(rows, off, col, val, B, 1.0, w=w) for w in (1, 2, 4, 8, 16, 32)}
    for w1, w2 in itertools.combinations(out, 2):
        assert not np.array_equal(out[w1], out[w2]), (w1, w2)
    # the same solve with each row's entries cut into contiguous runs per group: a wrong grouping the GPU tests would catch
    p = M.plan(rows, off, col)
    _, order, _ = M.levels(rows, p)
    Cc = np.zeros((rows, 3), np.float32)
    for i in order:
        b, e = p["t_off"][i], p["t_off"][i + 1]
        prod = val[p["t_vidx"][b:e]][:, None] * Cc[p["t_col"][b:e]]
        parts = [np.float32(0) * prod[0] if e > b else np.zeros(3, np.float32) for _ in range(32)]
        for g, chunk in enumerate(np.array_split(np.arange(e - b), 32)):
            s = np.zeros(3, np.float32)
            for m in chunk:
                s = s + prod[m]
            parts[g] = s
        s = np.array(parts)
        for o in (16, 8, 4, 2, 1):
            s = s + s[np.arange(32) ^ o]
        Cc[i] = (np.float32(1.0) * B[i] - s[0]) / val[p["diag_vidx"][i]]
    assert not np.array_equal(Cc, out[1])


def test_levels_on_hand_checked_patterns():
    off, col = M.SR.chain_pattern(50)
    for lower, tr in ((True, False), (False, False), (True, True)):
        lev, order, n = M.levels(50, M.plan(50, off, col, 0, lower, False, tr), lower, tr)
        assert n == 50                                             # every row is its own level
        assert np.array_equal(order, np.arange(50) if lower != tr else np.arange(49, -1, -1))
    off, col = M.SR.diagonal_pattern(37)
    lev, order, n = M.levels(37, M.plan(37, off, col))
    assert n == 1 and not lev.any() and np.array_equal(order, np.arange(37))
    for g in (3, 6, 9):
        off, col = M.SR.stencil5_pattern(g)
        for lower, tr in ((True, False), (False, False), (True, True), (False, True)):
            lev, order, n = M.levels(g * g, M.plan(g * g, off, col, 0, lower, False, tr), lower, tr)
            assert n == 2 * g - 1                                  # the anti-diagonals of the grid
            d = np.add.outer(np.arange(g), np.arange(g)).ravel()
            assert np.array_equal(lev, d if lower != tr else 2 * g - 2 - d)


def test_order_is_topological_and_sorted_by_level():
    for name, rows, off, col in M.fixtures():
        for lower, unit, tr in AXES:
            p = M.plan(rows, off, col, 0, lower, unit, tr)
            lev, order, n = M.levels(rows, p, lower, tr)
            assert sorted(order) == list(range(rows)) and np.all(np.diff(lev[order]) >= 0)
            pos = np.empty(rows, np.int64)
            pos[order] = np.arange(rows)
            i = np.repeat(np.arange(rows), np.diff(p["t_off"]))
            assert np.all(pos[p["t_col"]] < pos[i])              # a row is claimed after everything it depends on


def test_tile_function_matches_the_library(L):
    for nrhs in (1, 2, 3, 7, 8, 9, 31, 32, 33, 100, 128, 1000):
        for rm in (0, 1):
            assert L.b200spsm_csr_tile(nrhs, rm) == M.tile(nrhs, rm), (nrhs, rm)


# ---------------------------------------------------------------------------------------------------- routing
CSR, COO, SELL = 1, 4, 6
I32, I64 = 2, 3
F32, F64, F16, C32 = 0, 1, 2, 4


def route(lib, fmt=CSR, opa=0, opb=0, alg=0, off=I32, col=I32, a=F64, b=None, c=None, ct=None, fill=0, diag=0, rows=100, cols=None,
          nnz=500, nrhs=8, row_major=0, batch=1):
    b, c, ct = (a if v is None else v for v in (b, c, ct))
    cols = rows if cols is None else cols
    return lib.b200spsm_route(fmt, opa, opb, alg, off, col, a, b, c, ct, fill, diag, rows, cols, nnz, nrhs, row_major, batch)


def test_route_scope(L):
    for a, opa, opb, fill, diag, rm in itertools.product((F32, F64), (0, 1), (0, 1), (0, 1), (0, 1), (0, 1)):
        assert route(L, a=a, opa=opa, opb=opb, fill=fill, diag=diag, row_major=rm) >= 1
    assert route(L, fmt=COO) == 0 and route(L, fmt=SELL) == 0
    assert route(L, off=I64) == 0 and route(L, col=I64) == 0
    assert route(L, a=C32) == 0 and route(L, a=F16) == 0 and route(L, a=F32, b=F64, c=F64, ct=F64) == 0 and route(L, ct=F32) == 0
    assert route(L, opa=2) == 0 and route(L, opb=2) == 0 and route(L, alg=1) == 0
    assert route(L, fill=2) == 0 and route(L, diag=2) == 0 and route(L, cols=101) == 0
    assert route(L, batch=2) == 0 and route(L, nrhs=0) == 0
    assert route(L, rows=2 ** 31, nnz=5) == 0 and route(L, nnz=2 ** 31) == 0


def test_route_table(L):
    """No class was shown at parity with the closed library in a way the route can recognise (DESIGN.md 3.20): every call in
    scope, the measured shapes included, is forwarded (1)."""
    for a, rm, nrhs, opa, opb in itertools.product((F32, F64), (0, 1), (1, 2, 8, 31, 32, 100, 128, 1000), (0, 1), (0, 1)):
        for rows, per_row in ((490000, 3), (1 << 16, 2), (1 << 24, 1), (1 << 20, 9), (1 << 20, 8), (1 << 21, 9), (1 << 19, 9), (1, 1)):
            assert route(L, a=a, row_major=rm, nrhs=nrhs, opa=opa, opb=opb, rows=rows, nnz=per_row * rows) == 1, (a, rm, nrhs, rows)
    assert route(L, nrhs=2 ** 31 - 33) == 1 and route(L, nrhs=2 ** 31 - 32) == 0                # B200SPSM_MAX_NRHS


# ---------------------------------------------------------------------------------------------------- ABI
def test_header_declares_and_library_exports_every_spsm_symbol(L, built_lib):
    names = [n for n in declared_symbols() if n.startswith("b200spsm") or n.startswith("cusparseSpSM")]
    for n in ["cusparseSpSM_createDescr", "cusparseSpSM_destroyDescr", "cusparseSpSM_bufferSize", "cusparseSpSM_analysis",
              "cusparseSpSM_solve", "cusparseSpSM_updateMatrix", "b200spsm_csr_workspace_bytes", "b200spsm_csr_layout",
              "b200spsm_csr_analysis", "b200spsm_csr_solve", "b200spsm_csr_params", "b200spsm_route", "b200spsm_get_stats",
              "b200spsm_reset_stats"]:
        assert n in names, n
    have = exported(built_lib)
    assert not [n for n in names if n not in have]
    assert not [n for n in have if n.startswith("b200spsv") or n.startswith("cusparseSpSV")]


def test_spsv_library_exports_no_spsm():
    from cudalibrarysamples_b200 import build
    assert not [n for n in exported(build.SPSV_LIB_PATH) if "spsm" in n.lower()]


def test_layout(L):
    for rows, nnz, tr in ((0, 0, 0), (1, 1, 1), (1000, 4978, 0), (1000, 4978, 1), (64, 64, 0)):
        off = (ctypes.c_size_t * 10)()
        assert L.b200spsm_csr_layout(rows, nnz, tr, off) == 0
        o = list(off)[:9]
        assert o[0] == 0 and all(v % 256 == 0 for v in o) and o == sorted(o)
        assert o[1] - o[0] >= 16 and o[2] - o[1] >= 4 * rows and o[3] - o[2] >= 4 * (rows + 1) and o[4] - o[3] >= 4 * rows
        assert o[5] - o[4] >= 4 * nnz and o[6] - o[5] >= 4 * nnz and o[7] - o[6] >= 4 * rows
        assert o[8] - o[7] >= 4 * rows + (8 * nnz if tr else 0)
        assert L.b200spsm_csr_workspace_bytes(rows, nnz, tr) == o[8]
    assert L.b200spsm_csr_layout(-1, 0, 0, (ctypes.c_size_t * 10)()) == -1
    t, b = ctypes.c_int32(), ctypes.c_uint64()
    L.b200spsm_csr_params(ctypes.byref(t), ctypes.byref(b))
    assert t.value % 32 == 0 and t.value > 0 and 10 ** 9 <= b.value <= 60 * 10 ** 9


def test_host_side_argument_checks(L):
    ws = 1 << 20                                                   # never dereferenced: every call below fails first
    assert L.b200spsm_csr_analysis(None, -1, 0, None, None, 0, 1, 0, 0, ws, None, None) == -1
    assert L.b200spsm_csr_analysis(None, 4, 9, None, None, 0, 1, 0, 0, ws, None, None) == -1        # no arrays
    assert L.b200spsm_csr_analysis(None, 4, 9, ws, ws, 2, 1, 0, 0, ws, None, None) == -1            # base 2
    assert L.b200spsm_csr_analysis(None, 4, 9, ws, ws, 0, 1, 0, 0, None, None, None) == -1          # no workspace
    assert L.b200spsm_csr_analysis(None, 4, 9, ws, ws, 0, 1, 0, 0, ws + 4, None, None) == -1        # misaligned
    one = ctypes.c_double(1.0)
    a = ctypes.addressof(one)
    assert L.b200spsm_csr_solve(None, 7, 4, 9, 0, ws, None, a, 0, 2, ws, 1, 4, ws, 1, 4, ws) == -1    # dtype
    assert L.b200spsm_csr_solve(None, 1, 4, 9, 0, ws, None, None, 0, 2, ws, 1, 4, ws, 1, 4, ws) == -1  # alpha
    assert L.b200spsm_csr_solve(None, 1, 4, 9, 0, ws, None, a, 0, 2, None, 1, 4, ws, 1, 4, ws) == -1  # B
    assert L.b200spsm_csr_solve(None, 1, 4, 9, 0, ws, None, a, 0, 2, ws, 1, 4, None, 1, 4, ws) == -1  # C
    assert L.b200spsm_csr_solve(None, 1, 4, 9, 2, ws, None, a, 0, 2, ws, 1, 4, ws, 1, 4, ws) == -1    # unit
    assert L.b200spsm_csr_solve(None, 1, 4, 9, 0, ws, None, a, 0, -1, ws, 1, 4, ws, 1, 4, ws) == -1   # nrhs
    assert L.b200spsm_csr_solve(None, 1, 4, 9, 0, ws, None, a, 0, 2 ** 31 - 32, ws, 1, 4, ws, 1, 4, ws) == -1   # above the maximum
    assert L.b200spsm_csr_solve(None, 1, 4, 9, 0, ws, None, a, 0, 2, ws, 1, 4, ws, 1, 4, None) == -1  # workspace
    assert L.b200spsm_csr_solve(None, 1, 0, 0, 0, None, None, None, 0, 2, None, 1, 4, None, 1, 4, ws) == 0   # empty


# ---------------------------------------------------------------------------------------------------- bindings
def test_opt_in_sample_binds_spsm_to_the_spmv_library():
    from test_spsv_cpu import _bindings
    exe = os.path.join(ROOT, "oracle", "_ref", "spsm_csr_example.b200")
    if not os.path.exists(exe):
        pytest.skip("oracle/_ref not built (needs the reference checkout)")
    target = _bindings(exe)
    for s in ("cusparseSpSM_solve", "cusparseSpSM_analysis", "cusparseSpSM_bufferSize", "cusparseSpSM_createDescr"):
        assert "libb200spmv.so" in target(s), s
    assert "libcusparse.so.12" in target("cusparseCreate")
