"""CPU: the dispatch table of the shim's cusparseSpMV (csrc/cusparse_shim.cpp classify(), exported as b200spmv_route):
which calls run on the specialised kernels, which on spmv_generic.cu, which go to the closed library -- for every value of the
B200SPMV_GENERIC switch.  Pure host logic, no GPU.  Enum values: cusparse.h:4988-5007,5669-5676; library_types.h."""
import ctypes as C
import itertools

import pytest

from cudalibrarysamples_b200.lib import load

CSR, CSC, COO, BELL, BSR, SELL = 1, 2, 3, 5, 6, 7
N, T, H = 0, 1, 2
I32, I64, U16 = 2, 3, 1
F32, F64, F16, C32, C64, I8 = 0, 1, 2, 4, 5, 3
ALG_DEFAULT, COO_ALG2 = 0, 4
FORWARD, FAST, GENERIC = 0, 1, 2


@pytest.fixture()
def lib(built_lib):
    L = load(built_lib)
    yield L
    assert L.b200spmv_set_option(b"B200SPMV_GENERIC", b"csr") == 0      # back to the default


def route(L, fmt, op=N, alg=ALG_DEFAULT, off=I32, col=I32, a=F64, x=None, y=None, compute=None, rows=1000, cols=1000, nnz=16000):
    x = a if x is None else x
    y = x if y is None else y
    compute = x if compute is None else compute
    return L.b200spmv_route(fmt, op, alg, off, col, a, x, y, compute, C.c_int64(rows), C.c_int64(cols), C.c_int64(nnz))


@pytest.mark.parametrize("mode", [b"off", b"csr", b"all"])
def test_the_samples_calls_always_run_on_the_specialised_kernels(lib, mode):
    """spmv_csr / spmv_coo / spmv_sell / cg / bicgstab: int32 indices, one value type, NON_TRANSPOSE, ALG_DEFAULT."""
    assert lib.b200spmv_set_option(b"B200SPMV_GENERIC", mode) == 0
    for fmt, vt in itertools.product((CSR, COO, SELL), (F32, F64)):
        assert route(lib, fmt, a=vt) == FAST
    for fmt, op in itertools.product((CSR, COO), (T, H)):               # transposes of CSR / COO: specialised too
        assert route(lib, fmt, op=op) == FAST


@pytest.mark.parametrize("mode", [b"off", b"csr", b"all"])
def test_what_no_kernel_of_ours_takes_is_forwarded(lib, mode):
    assert lib.b200spmv_set_option(b"B200SPMV_GENERIC", mode) == 0
    for fmt in (CSC, BSR, BELL):
        assert route(lib, fmt) == FORWARD
    for vt in (F16, C32, C64, I8):
        assert route(lib, CSR, a=vt) == FORWARD
    assert route(lib, COO, alg=COO_ALG2) == FORWARD                        # the reproducibility promise stays with the closed library
    assert route(lib, CSR, a=F64, x=F32) == FORWARD                        # fp64 A with fp32 vectors: no such cuSPARSE combination
    assert route(lib, CSR, a=F32, x=F64, y=F32) == FORWARD                 # x / y / compute must agree
    assert route(lib, CSR, a=F32, x=F64, compute=F32) == FORWARD
    assert route(lib, CSR, off=I32, col=I64) == FORWARD
    assert route(lib, CSR, off=U16, col=U16) == FORWARD


def test_the_long_tail_by_switch(lib):
    tail_csr = [dict(off=I64, col=I64), dict(off=I64, col=I32), dict(a=F32, x=F64), dict(off=I64, col=I64, a=F32, x=F64, op=T),
                dict(rows=2**31 + 5, cols=2**31 + 5, off=I64, col=I64, nnz=2**33)]
    tail_other = [(COO, dict(off=I64, col=I64)), (COO, dict(a=F32, x=F64)), (COO, dict(off=I64, col=I64, op=T)),
                  (SELL, dict(off=I64, col=I64)), (SELL, dict(off=I64, col=I32)), (SELL, dict(op=T)), (SELL, dict(a=F32, x=F64, op=T))]
    want = {b"off": (FORWARD, FORWARD), b"csr": (GENERIC, FORWARD), b"all": (GENERIC, GENERIC)}
    for mode, (w_csr, w_other) in want.items():
        assert lib.b200spmv_set_option(b"B200SPMV_GENERIC", mode) == 0
        for kw in tail_csr:
            assert route(lib, CSR, **kw) == w_csr, (mode, kw)
        for fmt, kw in tail_other:
            assert route(lib, fmt, **kw) == w_other, (mode, fmt, kw)
