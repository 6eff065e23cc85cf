"""CPU: the numpy restatement of the incomplete LU / Cholesky factorizations (oracle/ilu0_ref.py) against textbook dense loops and
the pattern identities, and the host side of ilu0_csr.cu and the shim: exports and header, the workspace layout, argument rejection,
the route table and the B200SPMV_ILU0 option (DESIGN.md 3.26)."""
import ctypes as C
import os
import subprocess
import sys
import textwrap

import numpy as np
import pytest
import scipy.sparse as sp

from oracle import ilu0_ref as R
from oracle import oracle as O
from test_abi import declared_symbols, exported

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REAL = "/usr/local/cuda/lib64/libcusparse.so.12"
NEW = (["b200ilu0_workspace_bytes", "b200ilu0_layout", "b200ilu0_analysis", "b200ilu0_factor", "b200ilu0_zero_pivot", "b200ilu0_params",
        "b200ilu0_route", "cusparseCreateCsrilu02Info", "cusparseDestroyCsrilu02Info", "cusparseCreateCsric02Info",
        "cusparseDestroyCsric02Info", "cusparseXcsrilu02_zeroPivot", "cusparseXcsric02_zeroPivot"]
       + [f"cusparse{t}csrilu02_numericBoost" for t in "SDCZ"]
       + [f"cusparse{t}{k}{s}" for t in "SDCZ" for k in ("csrilu02", "csric02") for s in ("", "_bufferSize", "_bufferSizeExt", "_analysis")])


def random_pattern(n, density, seed, symmetric=True):
    A = sp.random(n, n, density=density, random_state=seed, format="csr")
    if symmetric:
        A = A + A.T
    A = A.tocsr()
    A.sort_indices()
    return R.with_diagonal(A.indptr, A.indices, n)


def dense_of(off, col, val, n):
    D = np.zeros((n, n), val.dtype)
    D[np.repeat(np.arange(n), np.diff(off)), col] = val
    return D


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("n,density,seed", [(1, 0.0, 1), (2, 1.0, 2), (9, 0.3, 3), (40, 0.15, 4), (64, 0.05, 5)])
def test_restatement_is_the_textbook_loop(n, density, seed, dtype):
    off, col = random_pattern(n, density, seed)
    val = R.dominant(off, col, dtype, seed)
    rowof = np.repeat(np.arange(n), np.diff(off))
    D = dense_of(off, col, val, n)
    for base in (0, 1):
        got, z = R.factor("lu", off + base, col + base, val, base)
        assert got.dtype == dtype and z == -1
        assert np.array_equal(got.view(np.uint8), R.dense_ilu0(D)[rowof, col].view(np.uint8))
        got, z = R.factor("ic", off + base, col + base, val, base)
        W = R.dense_ic0(np.tril(D))
        want = np.where(col <= rowof, W[rowof, col], val)
        assert z == -1 and np.array_equal(got.view(np.uint8), want.view(np.uint8))


@pytest.mark.parametrize("dtype,tol", [(np.float32, 2e-5), (np.float64, 1e-13)])
@pytest.mark.parametrize("name", ["stencil", "random", "unsymmetric"])
def test_pattern_identities(name, dtype, tol):
    """(L U)_ij = a_ij and (L L^T)_ij = a_ij on the stored pattern (of the lower triangle for IC)."""
    if name == "stencil":
        off, col, val = O.gen_stencil5(30, mass=0.3, ux=0.3, uy=0.2)
        val = val.astype(dtype)
    else:
        off, col = random_pattern(300, 0.02, 7, symmetric=name == "random")
        val = R.dominant(off, col, dtype, 8)
    n = off.size - 1
    rowof = np.repeat(np.arange(n), np.diff(off))
    A = dense_of(off, col, val.astype(np.float64), n)
    S = A != 0
    lu, _ = R.factor("lu", off, col, val)
    F = dense_of(off, col, lu.astype(np.float64), n)
    Lm, U = np.tril(F, -1) + np.eye(n), np.triu(F)
    assert np.abs((Lm @ U - A)[S]).max() <= tol * np.abs(A).max()
    ic, _ = R.factor("ic", off, col, val)
    Lc = np.tril(dense_of(off, col, ic.astype(np.float64), n))
    low = np.tril(S)
    assert np.abs((Lc @ Lc.T - A)[low]).max() <= tol * np.abs(A).max()
    up = col > rowof
    assert np.array_equal(ic[up], val[up])


def test_levels_of_the_cases():
    off, col = R.chain(100)
    assert R.levels(off, col).max() == 99
    off, col = R.diagonal(50)
    assert R.levels(off, col).max() == 0
    off, col, _ = O.gen_stencil5(20)
    assert R.levels(off, col).max() == 2 * 20 - 2


def test_zero_pivots_of_the_restatement():
    off, col = np.array([0, 2, 5, 7], np.int32), np.array([0, 1, 0, 1, 2, 1, 2], np.int32)
    val = np.array([2, 1, 4, 2, 1, 1, 3], np.float64)              # a_11 = 2 - (4 / 2) 1 = 0
    assert R.factor("lu", off, col, val)[1] == 1
    got, z = R.factor("lu", off, col, val, boost=True, tol=1e-8, boost_val=0.5)
    assert z == -1 and got[3] == 0.5
    val = np.array([1, 2, 2, 1, 0, 0, 2], np.float64)              # l_11^2 = 1 - 4 < 0
    assert R.factor("ic", off, col, val)[1] == 1



def test_structural_zeros_of_the_restatement():
    """A row without a stored diagonal is left as stored and reported; nothing is read from it, so a row that depends on it skips that
    step and is otherwise the factor of the same pattern with the dependency's diagonal present."""
    off, col = np.array([0, 2, 5, 7], np.int32), np.array([0, 1, 0, 1, 2, 1, 2], np.int32)
    val = np.array([4, 1, 1, 4, 1, 1, 4], np.float64)
    for kind in ("lu", "ic"):
        full, z = R.factor(kind, off, col, val)
        assert z == -1
        # row 1 without its diagonal: row 1 stays, row 2 skips its step on row 1
        o2, c2 = np.array([0, 2, 4, 6], np.int32), np.array([0, 1, 0, 2, 1, 2], np.int32)
        v2 = np.array([4, 1, 1, 1, 1, 4], np.float64)
        got, z = R.factor(kind, o2, c2, v2)
        assert z == 1 and np.array_equal(got[2:4], v2[2:4]) and got[4] == v2[4]
        assert got[5] == (4.0 if kind == "lu" else 2.0) and got[0] == full[0]
    got, z = R.factor("ic", np.array([0, 0, 0, 0]), np.array([], np.int32), np.array([], np.float64))
    assert z == 0 and got.size == 0


# ---- the library ------------------------------------------------------------------------------------------------------------
def test_header_declares_and_library_exports_the_factorization_symbols(built_lib):
    names, have = declared_symbols(), exported(built_lib)
    for n in NEW:
        assert n in names and n in have, n


def test_workspace_layout(built_lib):
    from cudalibrarysamples_b200.lib import load
    L = load(built_lib)
    up = lambda b: (b + 255) // 256 * 256      # noqa: E731
    for rows, nnz in ((0, 0), (1, 1), (490000, 2447200), (1 << 24, 1 << 24), (1000, 123457)):
        o = (C.c_size_t * 11)()
        assert L.b200ilu0_layout(rows, nnz, o) == 0
        sizes = [256, up(4 * rows), up(4 * rows), up(4 * (rows + 1)), up(4 * (rows + 1)), up(4 * nnz), up(4 * nnz), up(4 * (rows + 1)),
                 up(4 * rows)]
        assert list(o[:10]) == list(np.concatenate([[0], np.cumsum(sizes)]))
        assert L.b200ilu0_workspace_bytes(rows, nnz) == o[9]
    assert L.b200ilu0_layout(-1, 0, (C.c_size_t * 11)()) == -1 and L.b200ilu0_layout(1, 1, None) == -1
    assert L.b200ilu0_workspace_bytes(-1, 4) == 0
    t, c = C.c_int32(), C.c_int32()
    L.b200ilu0_params(C.byref(t), C.byref(c))
    assert t.value % 32 == 0 and c.value >= 1


def test_host_side_argument_rejection(built_lib):
    """-1 before any CUDA call, so no device is touched."""
    from cudalibrarysamples_b200.lib import load
    L = load(built_lib)
    buf = (C.c_double * 512)()
    a = C.addressof(buf) // 16 * 16 + 16
    assert L.b200ilu0_analysis(None, -1, 4, a, a, 0, a, None, None) == -1
    assert L.b200ilu0_analysis(None, 1 << 31, 4, a, a, 0, a, None, None) == -1
    assert L.b200ilu0_analysis(None, 4, 4, a, a, 2, a, None, None) == -1                 # base 2
    assert L.b200ilu0_analysis(None, 4, 4, a, a, 0, None, None, None) == -1              # no workspace
    assert L.b200ilu0_analysis(None, 4, 4, a, a, 0, a + 8, None, None) == -1             # workspace not 16-byte aligned
    assert L.b200ilu0_analysis(None, 4, 4, None, a, 0, a, None, None) == -1
    assert L.b200ilu0_analysis(None, 4, 4, a, None, 0, a, None, None) == -1
    f = lambda *x: L.b200ilu0_factor(None, *x)                                             # noqa: E731
    assert f(2, 0, 4, 4, a, a, 0, a, 0, None, None, 0, a) == -1                            # kind 2
    assert f(0, 2, 4, 4, a, a, 0, a, 0, None, None, 0, a) == -1                            # dtype 2
    assert f(0, 1, 4, 4, a, a, 0, a + 4, 0, None, None, 0, a) == -1                        # fp64 values on a 4-byte boundary
    assert f(0, 0, 4, 4, a, a, 0, a, 1, None, a, 0, a) == -1                               # boost without tol
    assert f(0, 0, 4, 4, a, a, 0, a, 1, a, None, 0, a) == -1                               # boost without boost_val
    assert f(0, 0, 4, 4, a, a, 0, None, 0, None, None, 0, a) == -1                         # no values
    assert f(0, 0, 4, 4, a, a, 0, a, 0, None, None, 0, a + 8) == -1                        # misaligned workspace
    assert f(1, 0, -4, 4, a, a, 0, a, 0, None, None, 0, a) == -1
    assert f(0, 0, 0, 0, None, None, 0, None, 0, None, None, 0, a) == 0                    # nothing to do, nothing launched
    pos = C.c_int()
    assert L.b200ilu0_zero_pivot(None, None, C.byref(pos), 0, None) == -1
    assert L.b200ilu0_zero_pivot(None, a, None, 0, None) == -1
    assert L.b200ilu0_zero_pivot(None, a, C.byref(pos), 2, None) == -1


ROUTE = textwrap.dedent(r"""
    import ctypes as C, os, sys
    sys.path.insert(0, os.path.dirname(os.path.dirname(sys.argv[1])))
    from cudalibrarysamples_b200.lib import load
    shim = load(sys.argv[1])
    mode = sys.argv[2]
    from scripts.ilu0_bench import native
    assert shim.b200spmv_set_option(b"B200SPMV_ILU0", b"sometimes") == -1
    if mode == "on":
        assert shim.b200spmv_set_option(b"B200SPMV_ILU0", b"on") == 0
        native = lambda *a: True
    for kind in (0, 1):
        for vt in (0, 1):
            for rows, nnz, levels in ((490000, 2447200, 1399), (490000, 2447200, 1), (1 << 16, 2 * (1 << 16) - 1, 1 << 16),
                                      (1 << 24, 1 << 24, 1), (1 << 20, 9 << 20, 40), (4096 * 4096, 5 * 4096 * 4096 - 4 * 4096, 8191),
                                      (10, 10, 1), (3, 7, 2)):
                want = 0 if mode == "forward" else int(native(kind, vt, rows, nnz, levels))
                assert shim.b200ilu0_route(kind, vt, rows, nnz, levels) == want, (kind, vt, rows, nnz, levels)
            # levels = 0: asked before analysis, whether any level count could be native (no class is measured native)
            assert shim.b200ilu0_route(kind, vt, 490000, 2447200, 0) == (0 if mode == "forward" else int(mode == "on"))
        for vt in (2, 4, 5, 14):                                            # 16-bit and complex types
            assert shim.b200ilu0_route(kind, vt, 1000, 5000, 10) == 0 and shim.b200ilu0_route(kind, vt, 1000, 5000, 0) == 0
        for rows, nnz, levels in ((0, 1, 1), (1, 0, 1), (4, 4, -1), (4, 4, 5), ((1 << 31), 4, 1), (4, (1 << 31), 1), (0, 1, 0)):
            assert shim.b200ilu0_route(kind, 1, rows, nnz, levels) == 0
    assert shim.b200ilu0_route(2, 1, 100, 100, 1) == 0 and shim.b200ilu0_route(-1, 1, 100, 100, 1) == 0
    if mode == "on":
        assert shim.b200spmv_set_option(b"B200SPMV_ILU0", b"auto") == 0
        assert shim.b200ilu0_route(0, 1, 1 << 24, 1 << 24, 1) == int(__import__("scripts.ilu0_bench").ilu0_bench.native(0, 1, 1 << 24, 1 << 24, 1))
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


def test_option_read_from_the_environment(built_lib):
    if not os.path.exists(REAL):
        pytest.skip("no toolkit libcusparse here")
    code = ("import os, sys; sys.path.insert(0, os.path.dirname(os.path.dirname(sys.argv[1]))); "
            "from cudalibrarysamples_b200.lib import load; s = load(sys.argv[1]); "
            "print(s.b200ilu0_route(0, 1, 1000, 5000, 1000))")
    for value, want in (("on", "1"), ("auto", None), ("", None)):
        env = {k: v for k, v in os.environ.items() if not k.startswith("B200SPMV_")}
        env.update(B200SPMV_CUSPARSE=REAL, B200SPMV_ILU0=value)
        p = subprocess.run([sys.executable, "-c", code, built_lib], capture_output=True, text=True, timeout=120, env=env)
        assert p.returncode == 0, p.stderr
        if want is not None:
            assert p.stdout.strip() == want
        else:
            sys.path.insert(0, ROOT)
            from scripts.ilu0_bench import native
            assert p.stdout.strip() == str(int(native(0, 1, 1000, 5000, 1000)))
