"""CPU: the format conversions of libb200spmv.so without a device -- symbols, the numpy restatement against scipy and the coosort
sample's golden arrays, the workspace formulas, host-side argument rejection and b200conv_route's table, B200SPMV_FORWARD included."""
import ctypes as C
import os
import subprocess
import sys
import textwrap

import numpy as np
import pytest
import scipy.sparse as sp

from cudalibrarysamples_b200.lib import load
from oracle import convert_ref as R
from oracle import oracle as O
from test_abi import declared_symbols, exported

REAL = "/usr/local/cuda/lib64/libcusparse.so.12"
NEW = ["b200csr2csc", "b200csr2csc_workspace_bytes", "b200coosort", "b200coosort_workspace_bytes", "b200coo2csr", "b200csr2coo",
       "b200identity_permutation", "b200conv_route", "cusparseCsr2cscEx2_bufferSize", "cusparseCsr2cscEx2",
       "cusparseXcoosort_bufferSizeExt", "cusparseXcoosortByRow", "cusparseXcoosortByColumn", "cusparseXcoo2csr", "cusparseXcsr2coo",
       "cusparseCreateIdentityPermutation"]


def test_header_declares_and_library_exports_the_conversion_symbols(built_lib):
    names = declared_symbols()
    have = exported(built_lib)
    for n in NEW:
        assert n in names and n in have, n


def _with_duplicates(rows, cols, nnz, seed):
    """a CSR pattern with repeated (row, col) entries and columns unsorted within each row"""
    rng = np.random.default_rng(seed)
    row = np.sort(rng.integers(0, rows, nnz))
    col = rng.integers(0, cols, nnz)
    off = np.concatenate([[0], np.cumsum(np.bincount(row, minlength=rows))])
    return off, col


def _patterns():
    off, col, _ = O.rmat_csr(2048, avg_nnz=16, seed=3, val_seed=4)
    yield "rmat", off, col, 2048, 2048
    off, col, _ = O.rmat_csr(1000, cols=70000, avg_nnz=8, seed=5, val_seed=6)
    yield "rmat_wide", off, col, 1000, 70000
    off, col, _ = O.gen_stencil5(23)
    yield "stencil5", off, col, len(off) - 1, len(off) - 1
    off, col = _with_duplicates(300, 40, 2000, 1)
    yield "duplicates_unsorted", off, col, 300, 40
    yield "no_entries", np.zeros(9, np.int64), np.zeros(0, np.int64), 8, 5


@pytest.mark.parametrize("base", [0, 1])
def test_csr2csc_restatement_matches_a_stable_sort(base):
    """scipy's tocsc() order is a stable sort of the entries by column; values follow their entries"""
    for name, off, col, rows, cols in _patterns():
        val = np.arange(len(col), dtype=np.float64) * 3 + 1
        ptr, ind, v = R.csr2csc(np.asarray(off) + base, np.asarray(col) + base, val, rows, cols, base)
        row = np.repeat(np.arange(rows), np.diff(off))
        o = np.argsort(np.asarray(col), kind="stable")
        assert np.array_equal(ind - base, row[o]) and np.array_equal(v, val[o]), name
        assert np.array_equal(ptr - base, np.searchsorted(np.asarray(col)[o], np.arange(cols + 1))), name
        if name != "duplicates_unsorted":                       # scipy's own CSC of a duplicate-free matrix
            T = sp.csr_matrix((val, np.asarray(col), np.asarray(off)), shape=(rows, cols)).tocsc()
            assert np.array_equal(ptr - base, T.indptr) and np.array_equal(ind - base, T.indices) and np.array_equal(v, T.data), name


def test_coosort_restatement_reproduces_the_sample():
    G = R.sample()
    rows, cols, P = R.coosort(G["rows"], G["columns"])
    assert rows.tolist() == G["rows_sorted"] and cols.tolist() == G["columns_sorted"] and P.tolist() == G["permutation"]
    assert (np.asarray(G["values"])[P]).tolist() == G["values_sorted"]


def test_coosort_restatement_orders_and_composes():
    rng = np.random.default_rng(2)
    rows, cols = rng.integers(0, 7, 500), rng.integers(0, 5, 500)
    P = rng.permutation(500)
    for by_row in (True, False):
        r, c, q = R.coosort(rows, cols, P, by_row)
        first, second = (r, c) if by_row else (c, r)
        key = first * 10 + second
        assert np.all(np.diff(key) >= 0)
        # sigma: P_out[i] = P_in[sigma(i)], and equal pairs keep their input order
        sigma = np.argsort(P)[q]
        assert np.array_equal(rows[sigma], r) and np.array_equal(cols[sigma], c)
        ties = np.diff(key) == 0
        assert np.all(np.diff(sigma)[ties] > 0)


@pytest.mark.parametrize("base", [0, 1])
def test_coo2csr_and_csr2coo_restatement(base):
    for name, off, col, rows, cols in _patterns():
        coo = R.csr2coo(np.asarray(off) + base, base)
        assert np.array_equal(coo - base, np.repeat(np.arange(rows), np.diff(off))), name
        assert np.array_equal(R.coo2csr(coo, rows, base), np.asarray(off) + base), name


def test_workspace_formulas(built_lib):
    lib = load(built_lib)
    for m, n, nnz in ((1000, 700, 5000), (5, 1, 4), (10, 10, 0), (1 << 20, 1 << 20, 16 << 20), (10 << 20, 10 << 20, 160 << 20), (0, 0, 0)):
        assert lib.b200csr2csc_workspace_bytes(m, n, nnz) == R.workspace("csr2csc", nnz)
        assert lib.b200coosort_workspace_bytes(m, n, nnz) == R.workspace("coosort", nnz)
        assert R.workspace("csr2csc", nnz) % 256 == 0 and R.workspace("coosort", nnz) % 256 == 0
    for f in (lib.b200csr2csc_workspace_bytes, lib.b200coosort_workspace_bytes):
        assert f(-1, 4, 4) == 0 and f(4, -1, 4) == 0 and f(4, 4, -1) == 0 and f(1 << 31, 4, 4) == 0 and f(4, 4, 1 << 31) == 0


def test_host_side_argument_rejection(built_lib):
    lib = load(built_lib)
    big = (C.c_byte * (1 << 20))()
    p = (C.addressof(big) + 255) // 256 * 256
    wsb = (1 << 20) - 256

    def csc(m=32, n=32, nnz=8, val=p, off=p, col=p, cval=p, cptr=p, cind=p, width=4, numeric=1, base=0, w=p, wb=wsb):
        return lib.b200csr2csc(None, m, n, nnz, val, off, col, cval, cptr, cind, width, numeric, base, w, wb)
    assert csc(m=-1) == -1 and csc(n=-1) == -1 and csc(nnz=-1) == -1 and csc(m=1 << 31) == -1 and csc(nnz=1 << 31) == -1
    assert csc(m=0) == -1 and csc(n=0) == -1                              # entries need a row and a column
    assert csc(base=2) == -1 and csc(width=3) == -1 and csc(width=32) == -1 and csc(width=0) == -1
    assert csc(off=None) == -1 and csc(col=None) == -1 and csc(cptr=None) == -1 and csc(cind=None) == -1
    assert csc(val=None) == -1 and csc(cval=None) == -1
    assert csc(off=p + 2) == -1 and csc(col=p + 1) == -1 and csc(cptr=p + 2) == -1 and csc(cind=p + 2) == -1
    assert csc(val=p + 4, width=8) == -1 and csc(cval=p + 8, width=16) == -1
    assert csc(w=None) == -1 and csc(w=p + 8) == -1 and csc(wb=100) == -1        # NULL, misaligned, short workspace

    def sort(by_row=1, m=32, n=32, nnz=8, rows=p, cols=p, P=p, w=p, wb=wsb):
        return lib.b200coosort(None, by_row, m, n, nnz, rows, cols, P, w, wb)
    assert sort(m=-1) == -1 and sort(n=-1) == -1 and sort(nnz=-1) == -1 and sort(m=1 << 31) == -1
    assert sort(rows=None) == -1 and sort(cols=None) == -1 and sort(P=None) == -1 and sort(rows=p + 2) == -1 and sort(P=p + 1) == -1
    assert sort(w=None) == -1 and sort(w=p + 4) == -1 and sort(wb=1000) == -1
    assert sort(nnz=0, rows=None, cols=None, P=None, w=None) == 0            # nothing to sort: no launch
    assert lib.b200coo2csr(None, p, 8, -1, p, 0) == -1 and lib.b200coo2csr(None, p, 8, 4, p, 2) == -1
    assert lib.b200coo2csr(None, None, 8, 4, p, 0) == -1 and lib.b200coo2csr(None, p, 8, 4, None, 0) == -1
    assert lib.b200coo2csr(None, p + 1, 8, 4, p, 0) == -1 and lib.b200coo2csr(None, p, -1, 4, p, 0) == -1
    assert lib.b200csr2coo(None, p, 8, 0, p, 0) == -1 and lib.b200csr2coo(None, p, 8, 4, p, -1) == -1
    assert lib.b200csr2coo(None, None, 8, 4, p, 0) == -1 and lib.b200csr2coo(None, p, 8, 4, None, 0) == -1
    assert lib.b200csr2coo(None, p, 8, 4, p + 2, 0) == -1 and lib.b200csr2coo(None, p, 0, 4, None, 0) == 0
    assert lib.b200identity_permutation(None, -1, p) == -1 and lib.b200identity_permutation(None, 8, None) == -1
    assert lib.b200identity_permutation(None, 8, p + 2) == -1 and lib.b200identity_permutation(None, 0, None) == 0


ROUTE = textwrap.dedent(r"""
    import ctypes as C, os, sys
    sys.path.insert(0, os.path.dirname(os.path.dirname(sys.argv[1])))     # the repository: argv[1] is its built library
    from cudalibrarysamples_b200.lib import load
    shim = load(sys.argv[1])
    forward = sys.argv[2] == "forward"
    native = eval(sys.argv[3])
    buf = (C.c_double * 64)()
    ok = C.addressof(buf) // 16 * 16 + 16
    CSR2CSC, ROW, COL, COO2CSR, CSR2COO, IDENTITY = range(6)
    shapes = [(1 << 20, 1 << 20, 16 << 20), (10 << 20, 10 << 20, 160 << 20), (2 << 20, 2 << 20, 32 << 20), (8192 ** 2, 8192 ** 2,
              5 * 8192 ** 2 - 4 * 8192), (4, 4, 11), (0, 0, 0), (100, 7, 0)]
    for m, n, nnz in shapes:
        for arg in (0, 1, 2, 4, 8, 16):
            want = 0 if forward else int(native(CSR2CSC, m, n, nnz, arg))
            assert shim.b200conv_route(CSR2CSC, m, n, nnz, arg, 1, ok) == want, (m, n, nnz, arg)
            assert shim.b200conv_route(CSR2CSC, m, n, nnz, arg, 2, ok) == 0              # only CUSPARSE_CSR2CSC_ALG1
            if nnz > 0:                                                                  # a NULL or misaligned buffer
                assert shim.b200conv_route(CSR2CSC, m, n, nnz, arg, 1, None) == 0
                assert shim.b200conv_route(CSR2CSC, m, n, nnz, arg, 1, ok + 8) == 0
        for arg in (-1, 3, 32):                                                          # a value type we do not move
            assert shim.b200conv_route(CSR2CSC, m, n, nnz, arg, 1, ok) == 0
        for op in (ROW, COL):
            assert shim.b200conv_route(op, m, n, nnz, 0, 0, ok) == (0 if forward else int(native(op, m, n, nnz, 0))), (op, m, n, nnz)
            if nnz > 0:
                assert shim.b200conv_route(op, m, n, nnz, 0, 0, None) == 0 and shim.b200conv_route(op, m, n, nnz, 0, 0, ok + 4) == 0
        for op in (COO2CSR, CSR2COO, IDENTITY):
            assert shim.b200conv_route(op, m, n, nnz, 0, 0, None) == (0 if forward else int(native(op, m, n, nnz, 0))), (op, m, n, nnz)
    for op in range(6):                                                                  # sizes past the sort's limits
        assert shim.b200conv_route(op, -1, 4, 4, 0, 1, ok) == 0 and shim.b200conv_route(op, 4, 4, -1, 0, 1, ok) == 0
        assert shim.b200conv_route(op, 4, 4, (1 << 31) - 65535, 0, 1, ok) == 0 and shim.b200conv_route(op, (1 << 31) - 63, 4, 4, 0, 1, ok) == 0
    assert shim.b200conv_route(6, 4, 4, 4, 0, 1, ok) == 0 and shim.b200conv_route(-1, 4, 4, 4, 0, 1, ok) == 0
    print("OK")
""")


@pytest.mark.parametrize("mode", ["default", "forward"])
def test_route_table(built_lib, mode):
    if not os.path.exists(REAL):
        pytest.skip("no toolkit libcusparse here")
    from scripts.convert_bench import NATIVE
    env = {k: v for k, v in os.environ.items() if not k.startswith("B200SPMV_")}
    env["B200SPMV_CUSPARSE"] = REAL
    if mode == "forward":
        env["B200SPMV_FORWARD"] = "1"
    p = subprocess.run([sys.executable, "-c", ROUTE, built_lib, mode, NATIVE], capture_output=True, text=True, timeout=600, env=env)
    assert p.returncode == 0 and p.stdout.strip().endswith("OK"), p.stdout + p.stderr
