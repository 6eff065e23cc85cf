"""CPU: the transposed CSR SpMM additions to libb200spmv.so without a device -- symbols, the numpy restatement of the transposed plan
against scipy's tocsc(), the workspace layout, host-side argument rejection, the routing table over real descriptors and the plan
trust of the side table."""
import ctypes as C
import os
import subprocess
import sys
import textwrap

import numpy as np
import pytest

from cudalibrarysamples_b200.lib import load
from oracle import oracle as O
from oracle import spmm_csr_t_ref as T
from test_abi import declared_symbols, exported

REAL = "/usr/local/cuda/lib64/libcusparse.so.12"
NEW = ["b200spmm_csr_t", "b200spmm_csr_t_plan", "b200spmm_csr_t_layout", "b200spmm_csr_t_workspace_bytes", "b200spmm_csr_t_route",
       "b200spmv_plan_trusted"]
F32, F64, F16, BF16 = 0, 1, 2, 14


def test_header_declares_and_library_exports_the_transposed_symbols(built_lib):
    names = declared_symbols()
    have = exported(built_lib)
    for n in NEW:
        assert n in names and n in have, n


def _random(rows, cols, nnz, seed):
    rng = np.random.default_rng(seed)
    flat = np.sort(rng.choice(rows * cols, nnz, replace=False))
    row, col = flat // cols, flat % cols
    off = np.concatenate([[0], np.cumsum(np.bincount(row, minlength=rows))])
    return off, col, rows, cols


def _patterns():
    off, col, _ = O.rmat_csr(4096, avg_nnz=16, seed=3, val_seed=4)
    yield "rmat", off, col, 4096, 4096
    off, col, _ = O.rmat_csr(3000, cols=70000, avg_nnz=8, seed=5, val_seed=6)      # three radix passes
    yield "rmat_wide", off, col, 3000, 70000
    off, col, _ = O.gen_stencil5(37)
    yield "stencil5", off, col, len(off) - 1, len(off) - 1
    yield "empty_rows_and_cols", *_random(50, 40, 60, 1)
    off, col, r, c = _random(300, 1, 120, 2)
    yield "one_column", off, col, r, c
    yield "no_entries", np.zeros(9, np.int64), np.zeros(0, np.int64), 8, 5
    yield "no_rows", np.zeros(1, np.int64), np.zeros(0, np.int64), 0, 5
    off, col, r, c = _random(1, 600, 500, 3)
    yield "one_long_row", off, col, r, c


@pytest.mark.parametrize("base", [0, 1])
def test_plan_restatement_matches_tocsc(base):
    for name, off, col, rows, cols in _patterns():
        off, col = np.asarray(off, np.int64) + base, np.asarray(col, np.int64) + base
        got = T.plan(off, col, cols, base)
        want = T.plan_scipy(off, col, rows, cols, base)
        for g, w, what in zip(got, want, ("tOff", "tRow", "perm")):
            assert np.array_equal(g, w), (name, what)


def test_radix_passes():
    assert [T.passes(c) for c in (0, 1, 2, 256, 257, 65536, 65537, 1 << 24, (1 << 24) + 1, (1 << 31) - 65)] == [1, 1, 1, 1, 2, 2, 3, 3, 4, 4]


def _shim(built_lib):
    lib = load(built_lib)
    return lib


@pytest.mark.parametrize("dtype", [F32, F64, F16, BF16])
def test_workspace_layout(built_lib, dtype):
    lib = _shim(built_lib)
    for rows, cols, n, nnz in ((1000, 700, 64, 5000), (5, 1, 3, 4), (10, 10, 32, 0), (1 << 20, 1 << 20, 256, 16 << 20), (0, 9, 8, 0)):
        for sbk, sbj in ((n, 1), (1, rows)):                       # op(B) row-major, column-major
            if dtype in (F16, BF16):
                prod = lib.b200spmm_csr16_workspace_bytes(rows, n, nnz, sbk, sbj)
            else:
                prod = lib.b200spmm_csr_workspace_bytes(dtype, rows, n, 1 if sbj == 1 else 0)
            want = T.layout(dtype, rows, cols, n, nnz, prod)
            offs = (C.c_size_t * 6)()
            total = lib.b200spmm_csr_t_layout(dtype, rows, cols, n, nnz, sbk, sbj, offs)
            assert total == want["total"] == lib.b200spmm_csr_t_workspace_bytes(dtype, rows, cols, n, nnz, sbk, sbj)
            assert list(offs) == [want[k] for k in ("t_off", "t_row", "perm", "scratch", "t_val", "ws")]
            assert all(o % 256 == 0 for o in offs)
            # the plan and its scratch depend on (cols, nnz) only
            other = (C.c_size_t * 6)()
            lib.b200spmm_csr_t_layout(F64 if dtype != F64 else F16, rows + 3, cols, n + 5, nnz, 1, 1, other)
            assert list(other)[:5] == list(offs)[:5]
    assert lib.b200spmm_csr_t_layout(3, 4, 4, 4, 4, 4, 1, None) == 0                    # unknown type
    assert lib.b200spmm_csr_t_layout(F32, 4, 4, 4, 17, 4, 1, None) == 0                 # more entries than the matrix holds
    assert lib.b200spmm_csr_t_layout(F32, -1, 4, 4, 0, 4, 1, None) == 0


def test_host_side_argument_rejection(built_lib):
    lib = _shim(built_lib)
    one = C.c_float(1.0)
    o = C.addressof(one)
    dummy = (C.c_int * 64)()
    p = C.addressof(dummy)
    big = (C.c_byte * (1 << 20))()
    ws = (C.addressof(big) + 255) // 256 * 256
    wsb = (1 << 20) - 256

    def call(dt=F32, ct=F32, rows=32, cols=32, n=8, nnz=2, off=p, col=p, val=p, base=0, alpha=o, beta=o, B=p, sbk=8, sbj=1, Cm=p, ldc=8,
             crow=1, w=ws, wb=wsb):
        return lib.b200spmm_csr_t(None, dt, ct, rows, cols, n, nnz, off, col, val, base, alpha, beta, 0, B, sbk, sbj, Cm, ldc, crow, 0, w, wb)
    assert call(dt=3, ct=3) == -1 and call(ct=F64) == -1 and call(dt=F16, ct=BF16) == -1 and call(dt=F16, ct=F64) == -1
    assert call(rows=-1) == -1 and call(cols=-1) == -1 and call(n=-1) == -1 and call(nnz=-1) == -1
    assert call(nnz=32 * 32 + 1) == -1 and call(rows=0, nnz=2) == -1
    assert call(base=2) == -1 and call(alpha=None) == -1 and call(beta=None) == -1
    assert call(sbk=-1) == -1 and call(sbj=-1) == -1
    assert call(sbk=8, sbj=2) == -1                                   # fp32 / fp64: op(B) neither row- nor column-major
    assert call(sbk=7) == -1 and call(sbk=1, sbj=31) == -1            # leading dimension of op(B) below the tight one
    assert call(ldc=7) == -1 and call(crow=0, ldc=31) == -1           # C is cols x n
    assert call(off=None) == -1 and call(col=None) == -1 and call(val=None) == -1 and call(B=None) == -1 and call(Cm=None) == -1
    assert call(w=None) == -1 and call(w=ws + 8) == -1 and call(wb=1000) == -1          # NULL, misaligned, short workspace
    assert call(rows=1 << 32, cols=1 << 32) == -1 and call(n=1 << 22) == -1 and call(dt=F16, ct=F16, n=32 * 65535 + 1) == -1
    assert call(cols=0, nnz=0) == 0 and call(n=0) == 0                # nothing to do: no launch
    plan = lambda rows=32, cols=32, nnz=2, off=p, col=p, base=0, w=ws, wb=wsb: lib.b200spmm_csr_t_plan(None, rows, cols, nnz, off, col,
                                                                                                       base, w, wb)
    assert plan(off=None) == -1 and plan(col=None) == -1 and plan(base=-1) == -1 and plan(nnz=32 * 32 + 1) == -1
    assert plan(w=None) == -1 and plan(w=ws + 4) == -1 and plan(wb=100) == -1


ROUTE = textwrap.dedent(r"""
    import ctypes as C, os, sys
    sys.path.insert(0, os.path.dirname(os.path.dirname(sys.argv[1])))     # the repository: argv[1] is its built library
    from cudalibrarysamples_b200.lib import load
    shim = load(sys.argv[1]); real = C.CDLL(sys.argv[2])
    I32, I64 = 2, 3
    F32, F64, F16, BF16, C32 = 0, 1, 2, 14, 4
    ROW, COL = 2, 1
    NT, TR, CT = 0, 1, 2
    DEFAULT, COO_ALG1, CSR_ALG1, CSR_ALG2, CSR_ALG3 = 0, 1, 4, 6, 12
    buf = (C.c_double * (1 << 20))()
    idx = (C.c_int * 4096)()
    ext = C.c_void_p(C.addressof(buf))

    def csr(rows, cols, nnz, vt=F32, it=I32, lib=shim, batch=1):
        d = C.c_void_p()
        assert lib.cusparseCreateCsr(C.byref(d), C.c_int64(rows), C.c_int64(cols), C.c_int64(nnz), idx, idx, buf, it, it, 0, vt) == 0
        if batch > 1:
            assert lib.cusparseCsrSetStridedBatch(d, batch, C.c_int64(0), C.c_int64(nnz)) == 0
        return d

    def dn(r, c, vt=F32, order=ROW, batches=1):
        d = C.c_void_p()
        assert real.cusparseCreateDnMat(C.byref(d), C.c_int64(r), C.c_int64(c), C.c_int64(c if order == ROW else r), buf, vt, order) == 0
        if batches > 1:
            assert real.cusparseDnMatSetStridedBatch(d, batches, C.c_int64(r * c)) == 0
        return d

    route = lambda a, b, c, opA=TR, opB=NT, ct=None, alg=DEFAULT, buffer=ext: shim.b200spmm_csr_t_route(
        a, b, c, opA, opB, ct if ct is not None else (F32 if vt in (F16, BF16) else vt), alg, buffer)
    native = eval(sys.argv[4])               # the measured classes: (trusted, opB, type, c type, n, rows, nnz, order B, order C) -> native
    forward = sys.argv[3] == "forward"
    m, k = 1 << 20, 1 << 20
    for vt, cvt in ((F32, F32), (F64, F64), (F16, F16), (F16, F32), (BF16, BF16), (BF16, F32)):
        for n in (8, 32, 64, 128, 256, 512):
            for per in (4, 16):
                for ob, oc in ((ROW, ROW), (COL, COL), (ROW, COL), (COL, ROW)):
                    a = csr(m, k, m * per, vt)
                    Cm = dn(k, n, cvt, oc)
                    for opB in (NT, TR):
                        B = dn(m, n, vt, ob) if opB == NT else dn(n, m, vt, ob)      # op(B) is m x n either way
                        for opA in (TR, CT):
                            r = route(a, B, Cm, opA=opA, opB=opB)
                            # a call without preprocess: the plan is not trusted
                            # opA = C: the closed library refuses it for real types
                            want = 0 if forward or opA == CT else int(native(False, opB, vt, cvt, n, m, m * per, ob, oc))
                            assert r == want, (vt, cvt, n, per, ob, oc, opA, opB, r)
                            assert route(a, B, Cm, opA=opA, opB=opB, buffer=None) == 0   # no buffer: forwarded
                        if opB == TR and not forward:
                            assert r == 0, (vt, n, per, ob, oc)                # opB = T was not measured: forwarded at every size
    if forward:
        print("OK"); sys.exit(0)
    for vt in (F32, F64, F16):
        a = csr(m, k, 4 * m, vt)
        B, Cm = dn(m, 64, vt, COL), dn(k, 64, vt, COL)
        assert route(a, B, Cm, opA=NT) == 0                                         # opA = N is not this route's
        for alg in (COO_ALG1, CSR_ALG2, CSR_ALG3):
            assert route(a, B, Cm, alg=alg) == 0, alg
        assert route(csr(m, k, 4 * m, vt, it=I64), B, Cm) == 0                     # 64-bit indices
        assert route(csr(m, k, 4 * m, vt, batch=4), dn(m, 64, vt, COL, 4), dn(k, 64, vt, COL, 4)) == 0   # strided batches
        assert route(None, B, Cm) == 0 and route(a, None, Cm) == 0
        assert route(a, dn(64, m, vt, ROW), Cm, opB=TR) == 0                       # not measured / fp32, fp64 opB = T
        # a fresh descriptor has no trusted plan of either kind, on any buffer
        assert shim.b200spmv_plan_trusted(a, ext, 0) == 0 and shim.b200spmv_plan_trusted(a, ext, 1) == 0
        assert shim.b200spmv_plan_trusted(a, None, 1) == 0 and shim.b200spmv_plan_trusted(None, ext, 1) == 0
    assert route(csr(m, k, 4 * m, C32), dn(m, 64, C32, COL), dn(k, 64, C32, COL), ct=C32) == 0   # complex
    # 16-bit with opA = T is no longer the csr16 route's question
    a = csr(m, k, 16 * m, F16)
    assert shim.b200spmm_csr16_route(a, dn(m, 64, F16, COL), dn(k, 64, F16, COL), TR, NT, F32, DEFAULT) == 0
    print("OK")
""")


def native_table():
    """the route's table (DESIGN.md 3.22), as the predicate the script evaluates"""
    from scripts.spmm_csr_t_bench import NATIVE
    return NATIVE


@pytest.mark.parametrize("mode", ["default", "forward"])
def test_route_table_over_real_descriptors(built_lib, mode):
    if not os.path.exists(REAL):
        pytest.skip("no toolkit libcusparse here")
    env = {k: v for k, v in os.environ.items() if not k.startswith("B200SPMV_")}
    env["B200SPMV_CUSPARSE"] = REAL
    if mode == "forward":
        env["B200SPMV_FORWARD"] = "1"
    p = subprocess.run([sys.executable, "-c", ROUTE, built_lib, REAL, mode, native_table()], capture_output=True, text=True, timeout=600,
                       env=env)
    assert p.returncode == 0 and p.stdout.strip().endswith("OK"), p.stdout + p.stderr
