"""CPU: the double-complex CSR SpMV additions to libb200spmv.so without a device -- symbols, the Gaussian-integer reference, the
correctly rounded fma and the fp64 restatement of the kernel's arithmetic, the route table (by shape and over real descriptors),
host-side argument rejection, workspace bytes and params."""
import ctypes as C
import os
import subprocess
import sys
import textwrap

import numpy as np
import pytest

from cudalibrarysamples_b200.lib import load
from oracle import spmv_csr_z_ref as R
from test_abi import declared_symbols, exported

REAL = "/usr/local/cuda/lib64/libcusparse.so.12"
NEW = ["b200spmv_csr_z", "b200spmv_csr_z_workspace_bytes", "b200spmv_csr_z_params"]
F32, F64, F16, BF16, C32, C64 = 0, 1, 2, 14, 4, 5
CSR, COO, SELL, CSC, BSR = 1, 2, 9, 3, 5
NT, TR, CT = 0, 1, 2
I32, I64 = 2, 3
DEFAULT, COO_ALG1, CSR_ALG1, CSR_ALG2, COO_ALG2, SELL_ALG1 = 0, 1, 2, 3, 4, 5
FORWARD, FAST, HALF16, ZCSR = 0, 1, 3, 4


def native():
    from scripts.spmv_csr_z_bench import NATIVE
    return eval(NATIVE)


def test_header_declares_and_library_exports_the_complex_spmv_symbols(built_lib):
    names = declared_symbols()
    have = exported(built_lib)
    for n in NEW:
        assert n in names and n in have, n


def test_fma_is_correctly_rounded():
    # 0.1 * 0.1 - 0.01: the unfused form rounds the product first and differs from the fused one
    assert R.fma(0.1, 0.1, -0.01) == 9.020562075079397e-19 and 0.1 * 0.1 - 0.01 != R.fma(0.1, 0.1, -0.01)
    e = 2.0 ** -30
    assert R.fma(1 + e, 1 + e, -1.0) == 2 * e + e * e                # exact: (1 + e)^2 - 1 keeps the e^2 term
    assert (1 + e) * (1 + e) - 1.0 == 2 * e                          # ... which the rounded product loses
    assert R.fma(1.0, 2.0 ** 53, 1.0) == 2.0 ** 53                   # ties to even
    assert R.fma(1.0, 2.0 ** 53, 3.0) == 2.0 ** 53 + 4
    assert str(R.fma(-0.0, 1.0, -0.0)) == "-0.0" and str(R.fma(0.0, -1.0, 0.0)) == "0.0" and str(R.fma(1.0, 1.0, -1.0)) == "0.0"
    assert np.isnan(R.fma(float("nan"), 1.0, 0.0)) and R.fma(float("inf"), 2.0, 1.0) == float("inf")


def test_complex_product_and_epilogue_forms():
    a, b = 0.1 + 0.7j, -0.3 + 0.9j
    p = R.cmul(a, b)
    assert p.real == R.fma(0.1, -0.3, -(0.7 * 0.9)) and p.imag == R.fma(0.1, 0.9, 0.7 * -0.3)
    acc, al, be, y = 1.1 - 2.3j, 0.75 + 0.5j, 0.5 - 0.25j, 3.0 + 1.0j
    t = R.cmul(be, y)
    out = R.epilogue(acc, al, be, y)
    assert out.real == R.fma(0.75, 1.1, R.fma(-0.5, -2.3, t.real)) and out.imag == R.fma(0.75, -2.3, R.fma(0.5, 1.1, t.imag))
    assert R.epilogue(acc, al, 0j, None) == complex(R.fma(0.75, 1.1, R.fma(-0.5, -2.3, 0.0)), R.fma(0.75, -2.3, R.fma(0.5, 1.1, 0.0)))


@pytest.mark.parametrize("base", [0, 1])
@pytest.mark.parametrize("op", ["N", "T", "C"])
def test_gaussian_integer_reference_matches_scipy(base, op):
    import scipy.sparse as sp
    lengths = [3, 0, 7, 1, 0, 12, 600]
    k = 700
    off, col = R.pattern(lengths, k, seed=1, base=base)
    val, x, y0 = R.values(len(lengths), k, len(col), seed=2)
    A = sp.csr_matrix((val, col - base, off - base), shape=(len(lengths), k))
    if op == "N":
        want = (2 - 1j) * (A @ x) + 1j * y0
        got = R.reference_int(off, col, val, x, y0, 2 - 1j, 1j, op, base)
    else:
        xt, yt = R.values(len(lengths), 0, 0, seed=3)[2], R.values(0, k, 0, seed=4)[1]
        At = A.T.conj() if op == "C" else A.T
        want = (2 - 1j) * (At @ xt) + 1j * yt
        got = R.reference_int(off, col, val, xt, yt, 2 - 1j, 1j, op, base, cols=k)
    assert np.array_equal(got, want)
    with pytest.raises(AssertionError):
        R.reference_int(off, col, val, x, y0, 0.5, 0, "N", base)                          # alpha not a Gaussian integer
    with pytest.raises(AssertionError):
        R.reference_int(off, col, val, np.full(k, 2.0 ** 52), y0, 1, 0, "N", base)       # sums past 2^53


def test_restatement_equals_the_integer_reference_on_gaussian_integers():
    E, Rn = 256, 8
    lengths = [0, 1, E - 1, E, E + 1, 0, 2 * E - 1, 2 * E + 1, 3, 40 * E + 17, 0]
    k = 50 * E
    off, col = R.pattern(lengths, k, seed=5)
    val, x, y0 = R.values(len(lengths), k, len(col), seed=6)
    for alpha, beta in ((1, 0), (2 - 1j, 1j), (-1j, -2)):
        assert np.array_equal(R.restate_n(off, col, val, x, y0, alpha, beta, E, Rn), R.reference_int(off, col, val, x, y0, alpha, beta))


def test_restatement_pins_the_summation_order():
    """one row of 2E + 3 entries: the first product is 2^53, every other 1.  A run is summed from 0 in order, so run 0 loses its seven
    ones to rounding while later runs are exact; a different order gives a different sum"""
    E, Rn = 256, 8
    n = 2 * E + 3
    val = np.ones(n, np.complex128)
    val[0] = 2.0 ** 53
    got = R.restate_n([0, n], np.zeros(n, np.int64), val, np.ones(1, np.complex128), None, 1, 0, E, Rn)
    # piece 0 = 2^53 + 31 runs of 8 = 2^53 + 248; piece 1 = 256; piece 2 = 3; each addition to 2^53 + ... rounds to even
    assert got[0].real == ((2.0 ** 53 + 248) + 256) + 3 and got[0].imag == 0
    assert got[0].real != 2.0 ** 53 + (n - 1)


def test_restatement_agrees_with_scipy_on_random_data():
    import scipy.sparse as sp
    lengths = [0, 1, 255, 256, 257, 511, 513, 5, 3000, 0, 17]
    k = 4000
    off, col = R.pattern(lengths, k, seed=7)
    rng = np.random.default_rng(8)
    val = rng.standard_normal(len(col)) + 1j * rng.standard_normal(len(col))
    x = rng.standard_normal(k) + 1j * rng.standard_normal(k)
    A = sp.csr_matrix((val, col, off), shape=(len(lengths), k))
    got = R.restate_n(off, col, val, x, None, 1, 0, 256, 8)
    bound = abs(A) @ np.abs(x)
    assert (np.abs(got - A @ x) <= (np.diff(off) + 4) * 4 * 2.0 ** -53 * bound + 1e-300).all()
    assert got[0] == 0 and got[9] == 0


def route(L, fmt=CSR, op=NT, alg=DEFAULT, off=I32, col=I32, a=C64, x=None, y=None, compute=None, rows=1 << 20, cols=1 << 20,
          nnz=16 << 20):
    x = a if x is None else x
    y = a if y is None else y
    compute = a if compute is None else compute
    return L.b200spmv_route(fmt, op, alg, off, col, a, x, y, compute, C.c_int64(rows), C.c_int64(cols), C.c_int64(nnz))


SHAPES = [(1 << 20, 16 << 20), (10 << 20, 160 << 20), (2 << 20, 32 << 20), (8192 * 8192, 5 * 8192 * 8192 - 4 * 8192),
          (256 ** 3, 7 * 256 ** 3 - 6 * 256 ** 2), (1000, 16000), (1 << 16, 1 << 20)]


@pytest.mark.parametrize("mode", [b"off", b"csr", b"all"])
def test_route_table(built_lib, mode):
    L = load(built_lib)
    assert L.b200spmv_set_option(b"B200SPMV_GENERIC", mode) == 0
    nat = native()
    for op in (NT, TR, CT):
        for rows, nnz in SHAPES:
            want = ZCSR if nat(op, rows, rows, nnz) else FORWARD
            for alg in (DEFAULT, CSR_ALG1, CSR_ALG2):
                assert route(L, op=op, alg=alg, rows=rows, cols=rows, nnz=nnz) == want, (op, rows, nnz, alg)
            # outside the class: forwarded whatever the shape
            ok = dict(op=op, rows=rows, cols=rows, nnz=nnz)
            assert route(L, a=C32, **ok) == FORWARD                                              # single complex
            assert route(L, a=C32, x=C64, y=C64, compute=C64, **ok) == FORWARD                   # mixed complex pairs
            assert route(L, a=F64, x=C64, y=C64, compute=C64, **ok) == FORWARD
            assert route(L, x=C32, y=C32, compute=C32, **ok) == FORWARD and route(L, compute=C32, **ok) == FORWARD
            assert route(L, y=C32, **ok) == FORWARD
            assert route(L, off=I64, col=I64, **ok) == FORWARD and route(L, col=I64, **ok) == FORWARD   # 64-bit indices
            for fmt in (COO, SELL, CSC, BSR):
                assert route(L, fmt=fmt, **ok) == FORWARD, fmt
            for alg in (COO_ALG1, COO_ALG2, SELL_ALG1):
                assert route(L, alg=alg, **ok) == FORWARD, alg
    assert route(L, rows=1 << 31, cols=1 << 20, nnz=16 << 31) == FORWARD                    # past int32
    # the tuples of the routing and 16-bit suites stay forwarded
    assert route(L, rows=1000, cols=1000, nnz=16000) == FORWARD and route(L, a=C32, rows=1000, cols=1000, nnz=16000) == FORWARD
    assert route(L, a=C32, rows=10 << 20, cols=10 << 20, nnz=160 << 20) == FORWARD
    # the fp32 / fp64 / 16-bit rows are unchanged
    assert route(L, a=F32) == FAST and route(L, a=F64) == FAST
    assert route(L, a=F32, op=TR) == FAST and route(L, a=F64, op=CT) == FAST
    assert route(L, a=F16, compute=F32, rows=10 << 20, cols=10 << 20, nnz=160 << 20) == HALF16
    assert route(L, a=BF16, y=F32, compute=F32, rows=10 << 20, cols=10 << 20, nnz=160 << 20) == FORWARD
    assert L.b200spmv_set_option(b"B200SPMV_GENERIC", b"csr") == 0


ROUTE = textwrap.dedent("""
    import ctypes as C, os, sys
    sys.path.insert(0, os.path.dirname(os.path.dirname(sys.argv[1])))     # the repository: argv[1] is its built library
    from cudalibrarysamples_b200.lib import load
    real = C.CDLL(sys.argv[2], mode=C.RTLD_GLOBAL)
    shim = load(sys.argv[1])
    I32, I64 = 2, 3
    F32, F64, C32, C64 = 0, 1, 4, 5
    buf = (C.c_double * 64)()
    idx = (C.c_int * 64)()

    def mat(rows, cols, nnz, vt=C64, it=I32, lib=shim, fmt="csr"):
        d = C.c_void_p()
        if fmt == "coo":
            assert lib.cusparseCreateCoo(C.byref(d), C.c_int64(rows), C.c_int64(cols), C.c_int64(nnz), idx, idx, buf, it, 0, vt) == 0
        elif fmt == "csc":
            assert lib.cusparseCreateCsc(C.byref(d), C.c_int64(rows), C.c_int64(cols), C.c_int64(nnz), idx, idx, buf, it, it, 0, vt) == 0
        else:
            assert lib.cusparseCreateCsr(C.byref(d), C.c_int64(rows), C.c_int64(cols), C.c_int64(nnz), idx, idx, buf, it, it, 0, vt) == 0
        return d

    def vec(n, vt, lib=shim):
        d = C.c_void_p()
        assert lib.cusparseCreateDnVec(C.byref(d), C.c_int64(n), buf, vt) == 0
        return d

    forward = sys.argv[3] == "forward"
    for rows, per in ((1000, 16), (1 << 20, 16), (2 << 20, 16), (10 << 20, 16), (1 << 20, 5)):
        nnz = rows * per
        a, x, y = mat(rows, rows, nnz), vec(rows, C64), vec(rows, C64)
        for op in (0, 1, 2):
            want = 0 if forward else shim.b200spmv_route(1, op, 0, I32, I32, C64, C64, C64, C64, rows, rows, nnz)
            for alg in (0, 2, 3):
                assert shim.b200spmv_csr16_route(a, x, y, op, C64, alg) == want, (rows, per, op, alg)
            assert shim.b200spmv_csr16_route(mat(rows, rows, nnz, lib=real), x, y, op, C64, 0) == want   # created behind our back
            assert shim.b200spmv_csr16_route(a, x, y, op, C64, 1) == 0                     # COO_ALG1
            assert shim.b200spmv_csr16_route(a, x, y, op, C32, 0) == 0                     # single-complex compute
            assert shim.b200spmv_csr16_route(mat(rows, rows, nnz, it=I64), x, y, op, C64, 0) == 0
            assert shim.b200spmv_csr16_route(mat(rows, rows, nnz, fmt="coo"), x, y, op, C64, 0) == 0
            assert shim.b200spmv_csr16_route(mat(rows, rows, nnz, fmt="csc", lib=real), x, y, op, C64, 0) == 0
            c32 = mat(rows, rows, nnz, vt=C32)
            assert shim.b200spmv_csr16_route(c32, vec(rows, C32), vec(rows, C32), op, C32, 0) == 0     # single complex
            assert shim.b200spmv_csr16_route(c32, x, y, op, C64, 0) == 0                                # mixed pair
            assert shim.b200spmv_csr16_route(a, x, vec(rows, C32), op, C64, 0) == 0
            assert shim.b200spmv_csr16_route(None, x, y, op, C64, 0) == 0
    # fp32 / fp64 descriptors keep their path
    n = 1 << 20
    want = 0 if forward else 1
    assert shim.b200spmv_csr16_route(mat(n, n, 16 * n, F32), vec(n, F32), vec(n, F32), 0, F32, 0) == want
    assert shim.b200spmv_csr16_route(mat(n, n, 16 * n, F64), vec(n, F64), vec(n, F64), 1, F64, 0) == want
    print("OK")
""")


@pytest.mark.parametrize("mode", ["default", "forward"])
def test_route_over_real_descriptors(built_lib, mode):
    if not os.path.exists(REAL):
        pytest.skip("no toolkit libcusparse here")
    env = {k: v for k, v in os.environ.items() if not k.startswith("B200SPMV_")}
    env["B200SPMV_CUSPARSE"] = REAL
    if mode == "forward":
        env["B200SPMV_FORWARD"] = "1"
    p = subprocess.run([sys.executable, "-c", ROUTE, built_lib, REAL, mode], capture_output=True, text=True, timeout=600, env=env)
    assert p.returncode == 0 and p.stdout.strip().endswith("OK"), p.stdout + p.stderr


def test_host_side_argument_rejection(built_lib):
    lib = load(built_lib)
    one = (C.c_double * 2)(1.0, 0.0)
    dummy = (C.c_double * 64)()
    p, o = (C.addressof(dummy) + 15) // 16 * 16, C.addressof(one)

    def call(op=0, m=32, k=32, nnz=2, off=p, col=p, val=p, base=0, alpha=o, beta=o, x=p, y=p):
        return lib.b200spmv_csr_z(None, op, m, k, nnz, off, col, val, base, alpha, beta, 0, x, y, None, 0)
    for op in (0, 1, 2):
        assert call(op, m=-1) == -1 and call(op, k=-1) == -1 and call(op, nnz=-1) == -1
        assert call(op, nnz=32 * 32 + 1) == -1                                                # more entries than the matrix holds
        assert call(op, base=2) == -1 and call(op, alpha=None) == -1 and call(op, beta=None) == -1
        assert call(op, off=None) == -1 and call(op, col=None) == -1 and call(op, val=None) == -1 and call(op, x=None) == -1
        assert call(op, y=None) == -1
        assert call(op, val=p + 8) == -1 and call(op, x=p + 8) == -1 and call(op, y=p + 8) == -1   # not 16-byte aligned
        assert call(op, m=1 << 31, k=1) == -1 and call(op, k=1 << 31) == -1 and call(op, m=1 << 20, k=1 << 20, nnz=1 << 31) == -1
    assert call(op=3) == -1 and call(op=-1) == -1
    assert call(0, m=0, nnz=0) == 0 and call(0, m=0, nnz=0, y=None, off=None) == 0              # nothing to do: no launch
    assert call(1, k=0, nnz=0) == 0 and call(2, k=0, nnz=0, y=None, off=None) == 0


def test_workspace_bytes_and_params(built_lib):
    lib = load(built_lib)
    P = R.params(lib)
    E = P["chunk"]
    assert E in (128, 256) and P["run"] == 8 and P["warps"] >= 1
    ws = lib.b200spmv_csr_z_workspace_bytes
    for rows, nnz in ((1 << 20, 16 << 20), (5, 1), (3, E), (3, E + 1), (7, 40 * E + 17)):
        assert ws(rows, nnz) == 2 * (-(-nnz // E)) * 16, (rows, nnz)
    assert ws(0, 0) == 0 and ws(10, 0) == 0 and ws(0, 10) == 0
