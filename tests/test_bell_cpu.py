"""CPU: the Blocked-ELL SpMM additions to libb200spmv.so without a device -- symbols, the reference samples' goldens, the int64
reference against scipy, the exactness precondition, the routing table over real descriptors, host-side argument rejection, and what
the kernels compile to."""
import ctypes as C
import os
import re
import subprocess
import sys
import textwrap

import numpy as np
import pytest

from cudalibrarysamples_b200.lib import load
from oracle import bell_ref as R
from test_abi import declared_symbols, exported

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REAL = "/usr/local/cuda/lib64/libcusparse.so.12"
NEW = ["b200spmm_bell", "b200spmm_bell_params", "b200spmm_bell_route", "cusparseSpMM", "cusparseSpMM_bufferSize", "cusparseSpMM_preprocess"]
F32, F16, BF16 = 0, 2, 14


def test_header_declares_and_library_exports_the_bell_symbols(built_lib):
    names = declared_symbols()
    have = exported(built_lib)
    for n in NEW:
        assert n in names and n in have, n
    assert "cusparseCreateBlockedEll" not in have            # the descriptor stays the closed library's


def test_spmm_blockedell_golden():
    E = R.samples()["spmm_blockedell"]
    B = np.array(E["B_colmajor"]).reshape(E["n"], E["ldb"]).T
    got = R.reference(E["rows"], E["cols"], E["bs"], E["col_ind"], np.array(E["values"]), B, None, E["alpha"], E["beta"])
    assert got.T.ravel().tolist() == E["C_result_colmajor"]
    assert got[0, 0] == 1 * 3 + 2 * 4 == 11                  # block-row 0 -> block column 1


def test_dense2sparse_blockedell_golden():
    D = R.samples()["dense2sparse_blockedell"]
    dense = np.array(D["dense_rowmajor"]).reshape(D["rows"], D["cols"])
    ci, v = R.from_dense(dense, D["bs"], D["ell_cols"])
    assert ci.ravel().tolist() == D["col_ind"] and v.ravel().tolist() == D["values"]     # -1 as the last slot of block-row 0
    assert np.array_equal(R.to_dense(D["rows"], D["cols"], D["bs"], D["col_ind"], D["values"]), dense)
    assert np.array_equal(R.to_scipy(D["rows"], D["cols"], D["bs"], D["col_ind"], D["values"]).toarray(), dense)


@pytest.mark.parametrize("bs", [1, 2, 4, 16])
@pytest.mark.parametrize("base", [0, 1])
def test_int64_reference_matches_scipy(bs, base):
    nbr, nbc, eb, n = 7, 6, 4, 9
    ci = R.structure(nbr, nbc, eb, [4, 0, 1, 3, 2], seed=bs, base=base)
    a, b, c0 = R.values(nbr * bs, eb * bs, nbc * bs, n, seed=3)
    sp = R.to_scipy(nbr * bs, nbc * bs, bs, ci, a, base)
    assert np.array_equal(R.products(nbr * bs, nbc * bs, bs, ci, a, b, base), (sp @ b.astype(np.float64)).astype(np.int64))
    got = R.reference(nbr * bs, nbc * bs, bs, ci, a, b, c0, -2.0, 0.5, base)
    assert np.array_equal(got, -2.0 * (sp @ b) + 0.5 * c0)
    assert (ci == -1).any(axis=1).sum() >= 3 and (ci == -1).all(axis=1).any()         # padding slots, and an all-empty block-row


def test_structure_puts_empty_slots_first_middle_and_last():
    ci = R.structure(64, 10, 5, [3], seed=1)
    assert (ci[:, 0] == -1).any() and (ci[:, -1] == -1).any() and (ci[:, 2] == -1).any()
    for row in ci:
        live = row[row != -1]
        assert len(live) == 3 and len(set(live.tolist())) == 3


def test_exactness_precondition():
    ci = R.structure(2, 3, 2, [2], seed=4)
    a, b, c0 = R.values(2 * 16, 2 * 16, 3 * 16, 5, seed=5)
    R.check_exact(32, 48, 16, ci, a, b, c0, 2.0, 0.5, "bf16")
    with pytest.raises(AssertionError):
        R.check_exact(32, 48, 16, ci, a, b, c0, 0.75, 0.0, "f32")                     # alpha not a power of two
    big = np.full_like(a, 9)
    with pytest.raises(AssertionError):
        R.check_exact(32, 48, 16, ci, big, np.full_like(b, 9), c0, 1.0, 0.0, "bf16")   # 2592 > 256: not exact in bf16
    R.check_exact(32, 48, 16, ci, big, np.full_like(b, 9), c0, 1.0, 0.0, "f32")


ROUTE = textwrap.dedent("""
    import ctypes as C, os, sys
    sys.path.insert(0, os.path.dirname(os.path.dirname(sys.argv[1])))     # the repository: argv[1] is its built library
    from cudalibrarysamples_b200.lib import load
    real = C.CDLL(sys.argv[2], mode=C.RTLD_GLOBAL)
    shim = load(sys.argv[1])
    I32, I64 = 2, 3
    F32, F64, F16, BF16, I8 = 0, 1, 2, 14, 3
    ROW, COL = 2, 1
    NT, TR = 0, 1
    buf = (C.c_double * 65536)()
    ci = (C.c_int * 64)()

    def bell(rows=64, cols=64, bs=16, ell=32, vt=F16, idx=I32):
        d = C.c_void_p()
        assert real.cusparseCreateBlockedEll(C.byref(d), C.c_int64(rows), C.c_int64(cols), C.c_int64(bs), C.c_int64(ell), ci, buf, idx,
                                             0, vt) == 0
        return d

    def dn(r, c, vt=F16, order=COL, batches=1):
        d = C.c_void_p()
        assert real.cusparseCreateDnMat(C.byref(d), C.c_int64(r), C.c_int64(c), C.c_int64(c if order == ROW else r), buf, vt, order) == 0
        if batches > 1:
            assert real.cusparseDnMatSetStridedBatch(d, batches, C.c_int64(r * c)) == 0
        return d

    route = lambda a, b, c, opA=NT, opB=NT, ct=F32, alg=0: shim.b200spmm_bell_route(a, b, c, opA, opB, ct, alg)
    A, B, Cm = bell(), dn(64, 8), dn(64, 8)
    if sys.argv[3] == "forward":
        assert route(A, B, Cm) == 0                                  # B200SPMV_FORWARD=1: everything to the closed library
        print("OK"); sys.exit(0)
    native = eval(sys.argv[4])                                       # the measured classes: (rows, cols, n, bs, order) -> native
    for bs in (2, 4, 16, 32, 64):
        for order in (COL, ROW):
            for vt, ct in ((F16, F16), (F16, F32), (BF16, BF16), (BF16, F32)):
                for rows, cols, n in ((64, 64, 8), (64, 64, 9), (64, 64, 128), (64, 64, 129), (128, 64, 8), (64, 128, 8),
                                      (16384, 16384, 512)):
                    r = route(bell(rows=rows, cols=cols, bs=bs, ell=bs, vt=vt), dn(cols, n, vt, order), dn(rows, n, ct, order))
                    assert r == int(native(rows, cols, n, bs, order)), (bs, order, vt, ct, rows, cols, n, r)
    assert route(A, dn(64, 8, order=ROW), Cm) == 0 and route(A, B, dn(64, 8, order=ROW)) == 0     # B and C in different orders
    assert route(A, B, Cm, alg=13) == 1                                        # CUSPARSE_SPMM_BLOCKED_ELL_ALG1
    assert route(A, B, Cm, alg=6) == 0                                         # a CSR algorithm
    assert route(A, B, Cm, opA=TR) == 0 and route(A, B, Cm, opB=TR) == 0      # transposes
    assert route(A, B, Cm, ct=F16) == 0                                        # 16-bit compute
    assert route(bell(vt=F32), dn(64, 8, F32), dn(64, 8, F32)) == 0            # fp32 Blocked-ELL
    assert route(bell(vt=I8), dn(64, 8, I8), dn(64, 8, F32)) == 0              # int8
    assert route(A, dn(64, 8, BF16), Cm) == 0                                  # A and B of different types
    assert route(bell(vt=BF16), dn(64, 8, BF16), dn(64, 8, F16)) == 0         # bf16 into an fp16 C
    assert route(A, dn(64, 8, batches=2), dn(64, 8, batches=2)) == 0          # strided batches
    assert route(A, dn(48, 8), Cm) == 1                                        # a shape mismatch stays native: rejected by the call
    csr = C.c_void_p()
    off = (C.c_int * 65)()
    assert shim.cusparseCreateCsr(C.byref(csr), C.c_int64(64), C.c_int64(64), C.c_int64(0), off, ci, buf, I32, I32, 0, F16) == 0
    assert route(csr, B, Cm) == 0                                              # not Blocked-ELL
    assert route(None, B, Cm) == 0 and route(A, None, Cm) == 0
    print("OK")
""")

# Classes routed natively (DESIGN.md 3.14): where the closed library measured faster, the call is forwarded
NATIVE = "lambda rows, cols, n, bs, order: rows <= 64 and cols <= 64 and n <= 128 and (bs == 16 or (bs == 2 and (order == COL or n <= 8)))"


@pytest.mark.parametrize("mode", ["default", "forward"])
def test_route_table_over_real_descriptors(built_lib, mode):
    if not os.path.exists(REAL):
        pytest.skip("no toolkit libcusparse here")
    env = {k: v for k, v in os.environ.items() if not k.startswith("B200SPMV_")}
    env["B200SPMV_CUSPARSE"] = REAL
    if mode == "forward":
        env["B200SPMV_FORWARD"] = "1"
    p = subprocess.run([sys.executable, "-c", ROUTE, built_lib, REAL, mode, NATIVE], capture_output=True, text=True, timeout=120, env=env)
    assert p.returncode == 0 and p.stdout.strip().endswith("OK"), p.stdout + p.stderr


def test_host_side_argument_rejection(built_lib):
    lib = load(built_lib)
    one = C.c_float(1.0)
    dummy = (C.c_int * 64)()
    p = C.addressof(dummy)

    def call(at=F16, ct=F16, rows=32, cols=32, n=8, bs=16, ell=32, ci=p, v=p, base=0, alpha=C.addressof(one), beta=C.addressof(one), B=p,
             ldb=32, brow=0, Cp=p, ldc=32, crow=0):
        return lib.b200spmm_bell(None, at, ct, rows, cols, n, bs, ell, ci, v, base, alpha, beta, 0, B, ldb, brow, Cp, ldc, crow)
    assert call(at=F32) == -1 and call(at=BF16, ct=F16) == -1 and call(ct=1) == -1
    assert call(rows=-1) == -1 and call(n=-1) == -1 and call(bs=0) == -1
    assert call(rows=24) == -1 and call(cols=24) == -1 and call(ell=24) == -1   # not multiples of bs
    assert call(ell=48) == -1                                                    # more slots than block columns
    assert call(base=2) == -1 and call(alpha=None) == -1 and call(beta=None) == -1
    assert call(ldb=31) == -1 and call(ldc=31) == -1
    assert call(brow=1, ldb=7) == -1 and call(crow=1, ldc=7) == -1
    assert call(ci=None) == -1 and call(v=None) == -1 and call(B=None) == -1 and call(Cp=None) == -1
    assert call(rows=0) == 0 and call(n=0) == 0                                  # nothing to do: no launch
    assert call(rows=1 << 32, cols=1 << 32, ell=32) == -1


def test_params(built_lib):
    P = R.params(load(built_lib))
    assert P["n_tile"] % 16 == 0 and P["stages"] >= 2 and P["max_rows_per_cta"] % 16 == 0


def test_sass_of_the_bell_kernels(built_lib):
    """the tensor path runs HMMA fed by LDSM (ldmatrix, .T for a row-major B) from LDGSTS (cp.async); the scalar path has no tensor
    instruction; no kernel spills to local memory"""
    sass = subprocess.check_output(["cuobjdump", "-sass", built_lib], text=True)

    def kernel_sass(_, pattern):
        m = re.search(r"Function : \S*" + pattern + r".*?(?=Function :|\Z)", sass, re.S)
        assert m, pattern
        return m.group(0)
    for t in ("6__half", "13__nv_bfloat16"):
        for bm in (16, 32, 64):
            for brow in (0, 1):
                body = kernel_sass(built_lib, rf"bell_mma_kernelI{t}Li{bm}ELb{brow}E")
                assert "HMMA.16816.F32" in body and "LDGSTS" in body and "LDSM" in body, (t, bm, brow)
                assert ("LDSM.16.MT88" in body) == bool(brow), (t, bm, brow)
                assert "STL" not in body
        for rf in (0, 1):
            body = kernel_sass(built_lib, rf"bell_scalar_kernelI{t}Lb{rf}E")
            assert "HMMA" not in body and "STL" not in body
    assert "HMMA.16816.F32.BF16" in kernel_sass(built_lib, r"bell_mma_kernelI13__nv_bfloat16Li64ELb0E")
