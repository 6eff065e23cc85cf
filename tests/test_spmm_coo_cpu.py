"""CPU: the COO SpMM additions to libb200spmv.so without a device -- symbols, the samples' goldens, the int64 reference against scipy,
the exactness precondition, the numpy model of the chunk / run / carry walk at the GPU test sizes, the routing table over real
descriptors, cusparseCooSetStridedBatch, host-side argument rejection, and what the kernels compile to."""
import ctypes as C
import os
import re
import subprocess
import sys
import textwrap

import numpy as np
import pytest
import scipy.sparse as sp

from oracle import oracle as O
from oracle import spmm_coo_ref as R
from test_abi import declared_symbols, exported

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REAL = "/usr/local/cuda/lib64/libcusparse.so.12"
NEW = ["b200spmm_coo", "b200spmm_coo_workspace_bytes", "b200spmm_coo_params", "b200spmm_coo_route", "cusparseCooSetStridedBatch"]


def test_header_declares_and_library_exports_the_coo_spmm_symbols(built_lib):
    names = declared_symbols()
    have = exported(built_lib)
    for n in NEW:
        assert n in names and n in have, n


def test_spmm_coo_goldens():
    S = R.samples()
    Q = S["spmm_coo"]
    B = np.asarray(Q["B"]).reshape(Q["n"], 4).T
    got = R.reference(4, 4, Q["row"], Q["col"], Q["val"], B, None, 1.0, 0.0)
    assert got.T.ravel().tolist() == list(Q["C"]) == O.TOY["spmm_C"].T.ravel().tolist()
    Q = S["spmm_coo_batched"]
    for i in range(2):
        sl = slice(9 * i, 9 * i + 9)
        B = np.asarray(Q["B"][12 * i:12 * i + 12]).reshape(3, 4).T
        got = R.reference(4, 4, Q["row"][sl], Q["col"][sl], Q["val"][sl], B, None, 1.0, 0.0)
        assert got.T.ravel().tolist() == O.TOY_BATCHED["C"][i].tolist()


@pytest.mark.parametrize("base", [0, 1])
@pytest.mark.parametrize("transpose", [False, True])
def test_int64_reference_matches_scipy(base, transpose):
    rng = np.random.default_rng(3)
    rows, cols, nnz, n = 30, 20, 150, 7
    row, col = rng.integers(0, rows, nnz), rng.integers(0, cols, nnz)          # unsorted, with duplicates
    v, b, c0 = R.values(nnz, rows if transpose else cols, cols if transpose else rows, n, seed=4)
    A = sp.coo_matrix((v.astype(np.float64), (row, col)), shape=(rows, cols))
    opA = A.T if transpose else A
    got = R.reference(rows, cols, row + base, col + base, v, b, c0, -2.0, 0.5, base, transpose)
    assert np.array_equal(got, -2.0 * (opA @ b) + 0.5 * c0)
    assert np.array_equal(R.products(rows, cols, row + base, col + base, v, b, base, transpose), (opA @ b).astype(np.int64))


def test_exactness_precondition():
    row = R.sorted_rows(4, [3, 0, 2, 1])
    v, b, c0 = R.values(6, 5, 4, 3, seed=5)
    col = np.array([0, 1, 2, 3, 4, 0])
    R.check_exact(4, 5, row, col, v, b, c0, 2.0, 0.5)
    with pytest.raises(AssertionError):
        R.check_exact(4, 5, row, col, v, b, c0, 0.75, 0.0)                    # alpha not a power of two
    with pytest.raises(AssertionError):
        R.check_exact(4, 5, row, col, np.full(6, 1 << 12), np.full_like(b, 1 << 12), c0, 1.0, 0.0)     # partial sums past 2^24


def gpu_structures(chunk):
    """the row structures tests/test_spmm_coo_gpu.py runs (its structures() helper)"""
    src = open(os.path.join(ROOT, "tests", "test_spmm_coo_gpu.py")).read()
    body = src[src.index("def structures(chunk):"):]
    body = body[:body.index("\n\n\n")]
    ns = {}
    exec(body, {"np": np, "R": R}, ns)
    return ns["structures"](chunk)


def test_chunk_walk_model_at_the_gpu_test_sizes(built_lib):
    """the numpy restatement of the sorted path computes the reference and writes every entry of C once, and the GPU test structures
    reach every edge of the walk"""
    chunk = R.params(C.CDLL(built_lib))["chunk"]
    seen = {}
    for name, (rows, row) in gpu_structures(chunk).items():
        v, b, c0 = R.values(row.size, 37, rows, 5, seed=len(name))
        col = np.random.default_rng(len(name)).integers(0, 37, row.size)
        for alpha, beta in ((2.0, -1.0), (1.0, 0.0)):
            out, writes = R.walk(rows, row, col, v, b, c0, alpha, beta, chunk)
            assert np.array_equal(out, R.reference(rows, 37, row, col, v, b, c0, alpha, beta)), name
            assert (writes == 1).all(), name
        e = R.edges(rows, row, chunk)
        for k, x in e.items():
            seen.setdefault(k, set()).add(x)
    assert {chunk - 1, 0, 1} <= seen["nnz_mod"]                                   # nnz at chunk - 1, chunk, chunk + 1
    assert max(seen["max_span"]) >= 4 and 2 in seen["max_span"]                   # a row across two chunks and across every chunk
    for k in ("empty_first", "empty_last", "empty_middle", "empty_across_border"):
        assert True in seen[k], k
    out, writes = R.walk(7, np.zeros(0, np.int64), [], [], np.zeros((5, 3)), np.ones((7, 3)), 1.0, 0.5, chunk)
    assert (out == 0.5).all() and (writes == 1).all()                             # all rows empty, nnz = 0


ROUTE = textwrap.dedent("""
    import ctypes as C, sys
    real = C.CDLL(sys.argv[2], mode=C.RTLD_GLOBAL)
    shim = C.CDLL(sys.argv[1])
    shim.b200spmm_coo_route.argtypes = [C.c_void_p] * 3 + [C.c_int] * 4
    I32, I64 = 2, 3
    F32, F64, F16 = 0, 1, 2
    ROW, COL = 2, 1
    NT, TR = 0, 1
    buf = (C.c_double * 65536)()
    idx = (C.c_int64 * 4096)()

    M = 1 << 16                                                      # the smallest matrix measured at parity
    def coo(rows=M, cols=48, nnz=16 * M, vt=F32, it=I32, batch=1, stride=16 * M, via=shim):
        d = C.c_void_p()
        assert via.cusparseCreateCoo(C.byref(d), C.c_int64(rows), C.c_int64(cols), C.c_int64(nnz), idx, idx, buf, it, 0, vt) == 0
        if batch > 1:
            assert via.cusparseCooSetStridedBatch(d, batch, C.c_int64(stride)) == 0
        return d

    def dn(r, c, vt=F32, order=COL, batches=1, stride=None):
        d = C.c_void_p()
        assert real.cusparseCreateDnMat(C.byref(d), C.c_int64(r), C.c_int64(c), C.c_int64(c if order == ROW else r), buf, vt, order) == 0
        if batches > 1:
            assert real.cusparseDnMatSetStridedBatch(d, batches, C.c_int64(r * c if stride is None else stride)) == 0
        return d

    route = lambda a, b, c, opA=NT, opB=NT, ct=F32, alg=0: shim.b200spmm_coo_route(a, b, c, opA, opB, ct, alg)
    A, B, Cm = coo(), dn(48, 32), dn(M, 32)
    if sys.argv[3] == "forward":
        assert route(A, B, Cm) == 0                                  # B200SPMV_FORWARD=1: everything to the closed library
        print("OK"); sys.exit(0)
    native = eval(sys.argv[4])                                       # the measured classes: (dtype, opA, order, n) -> native
    for vt in (F32, F64):
        for op in (NT, TR):
            for order in (COL, ROW):
                for n in (8, 32, 64, 128, 129, 512):
                    kr, cr = (48, M) if op == NT else (M, 48)
                    r = route(coo(vt=vt), dn(kr, n, vt, order), dn(cr, n, vt, order), opA=op, ct=vt)
                    assert r == int(native(vt, op, order, n)), (vt, op, order, n, r)
    for alg in (0, 1, 3, 5):                                         # DEFAULT, COO_ALG1, COO_ALG3, COO_ALG4
        assert route(A, B, Cm, alg=alg) == int(native(F32, NT, COL, 32)), alg
    assert route(A, B, Cm, alg=2) == 0                               # COO_ALG2: bit-wise reproducible, forwarded
    assert route(A, B, Cm, alg=6) == 0                               # a CSR algorithm
    assert route(A, B, Cm, opB=TR) == 0 and route(A, B, Cm, opA=2) == 0
    assert route(coo(it=I64), B, Cm) == 0                            # 64-bit indices
    assert route(coo(vt=F16), dn(48, 32, F16), dn(M, 32, F16), ct=F32) == 0      # fp16
    assert route(A, dn(48, 32, F64), dn(M, 32, F64), ct=F64) == 0    # mixed types
    assert route(A, B, Cm, ct=F64) == 0
    # strided batches: A strided, A broadcast (stride 0), B shared (batch count 1); the count and the stride reach the side table
    Ab = coo(batch=3)
    cnt = C.c_int()
    assert real.cusparseSpMatGetStridedBatch(Ab, C.byref(cnt)) == 0 and cnt.value == 3          # the real descriptor keeps it
    assert route(Ab, dn(48, 32, batches=3), dn(M, 32, batches=3)) == 3
    assert route(coo(batch=3, stride=0), dn(48, 32, batches=3), dn(M, 32, batches=3)) == 3
    assert route(Ab, B, dn(M, 32, batches=3)) == 3
    assert route(Ab, dn(48, 32, batches=2), dn(M, 32, batches=3)) == 0                          # batch counts disagree
    assert route(coo(batch=3, via=real), dn(48, 32, batches=3), dn(M, 32, batches=3)) == 0     # batch set behind the shim's back
    assert route(A, dn(40, 32), Cm) == 1                            # a shape mismatch stays native: rejected by the call
    assert route(coo(nnz=16 * M - 1), B, Cm) == 0                   # fewer than 16 entries per row on average (Laplace 7-pt: slower)
    assert route(coo(rows=M - 1, nnz=16 * M), B, dn(M - 1, 32)) == 0                            # smaller than any class measured
    assert route(A, B, dn(M, 32, order=ROW)) == 0 and route(A, dn(48, 32, order=ROW), Cm) == 0  # row-major or mixed orders
    csr = C.c_void_p()
    off = (C.c_int * 65)()
    assert shim.cusparseCreateCsr(C.byref(csr), C.c_int64(64), C.c_int64(48), C.c_int64(0), off, idx, buf, I32, I32, 0, F32) == 0
    assert route(csr, B, Cm) == 0                                   # not COO
    assert route(None, B, Cm) == 0 and route(A, None, Cm) == 0
    print("OK")
""")

# Classes routed natively (DESIGN.md 3.15): (value type, opA, order of B and C, n) -> native
NATIVE = "lambda vt, op, order, n: op == NT and order == COL and 32 <= n <= 128"


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
    lib = C.CDLL(built_lib)
    vp, i64 = C.c_void_p, C.c_int64
    lib.b200spmm_coo.argtypes = [vp, C.c_int, C.c_int, i64, i64, i64, i64, vp, vp, vp, C.c_int32, vp, vp, C.c_int, vp, i64, C.c_int, vp, i64,
                                 C.c_int, C.c_int, i64, i64, i64, vp, C.c_size_t]
    one = C.c_float(1.0)
    dummy = (C.c_int * 64)()
    p = C.addressof(dummy)

    def call(dt=0, tr=0, rows=8, cols=6, n=4, nnz=5, row=p, col=p, val=p, base=0, alpha=C.addressof(one), beta=C.addressof(one), B=p, ldb=6,
             brow=0, Cp=p, ldc=8, crow=0, batch=1, a_stride=0, b_stride=0, c_stride=0):
        return lib.b200spmm_coo(None, dt, tr, rows, cols, n, nnz, row, col, val, base, alpha, beta, 0, B, ldb, brow, Cp, ldc, crow, batch,
                                a_stride, b_stride, c_stride, None, 0)
    assert call(dt=2) == -1 and call(rows=-1) == -1 and call(n=-1) == -1 and call(nnz=-1) == -1
    assert call(base=2) == -1 and call(alpha=None) == -1 and call(beta=None) == -1
    assert call(ldb=5) == -1 and call(ldc=7) == -1 and call(brow=1, ldb=3) == -1 and call(crow=1, ldc=3) == -1
    assert call(tr=1) == -1                                                                                    # A^T: B is rows x n
    assert call(tr=1, ldb=7, ldc=6) == -1 and call(tr=1, ldb=8, ldc=5) == -1
    assert call(row=None) == -1 and call(col=None) == -1 and call(val=None) == -1 and call(B=None) == -1 and call(Cp=None) == -1
    assert call(batch=0) == -1 and call(batch=65536) == -1 and call(a_stride=-1) == -1
    assert call(batch=2, c_stride=8 * 4 - 1) == -1                                                             # overlapping outputs
    assert call(rows=0) == -1                                                                                  # entries in an empty A
    assert call(rows=0, nnz=0) == 0 and call(n=0) == 0                                                         # nothing to do: no launch
    assert call(rows=1 << 32) == -1 and call(nnz=1 << 31) == -1 and call(n=64 * 65535 + 1, ldb=1 << 23, brow=1) == -1


def test_params_and_workspace(built_lib):
    lib = C.CDLL(built_lib)
    P = R.params(lib)
    assert P["chunk"] % 32 == 0 and P["panel"] == 64 and P["flag_offset"] == 0
    lib.b200spmm_coo_workspace_bytes.restype = C.c_size_t
    lib.b200spmm_coo_workspace_bytes.argtypes = [C.c_int, C.c_int] + [C.c_int64] * 4 + [C.c_int, C.c_int, C.c_int64]
    ws = lambda *a: lib.b200spmm_coo_workspace_bytes(*a)          # noqa: E731
    small = ws(0, 0, 100, 80, 8, 1000, 1, 1, 0)
    assert small > 0 and small % 256 == 0
    assert ws(0, 0, 100, 80, 8, 1000, 0, 1, 0) >= small + 80 * 8 * 4                 # + the row-major copy of a column-major B
    assert ws(0, 0, 100, 80, 2, 1000, 0, 1, 0) == ws(0, 0, 100, 80, 2, 1000, 1, 1, 0)   # n < 4: B read in place
    assert ws(1, 0, 100, 80, 8, 1000, 1, 1, 0) > small and ws(0, 0, 100, 80, 8, 1000, 1, 3, 0) > small
    assert ws(0, 1, 100, 80, 8, 1000, 0, 1, 0) >= ws(0, 0, 100, 80, 8, 1000, 1, 1, 0) + 100 * 8 * 4     # A^T: B has `rows` rows
    assert ws(2, 0, 100, 80, 8, 1000, 1, 1, 0) == 0


def test_sass_of_the_coo_spmm_kernels(built_lib):
    """the sorted path (check, sorted, fix-up kernels) has no atomics; the atomic path adds with RED / ATOM; nothing spills"""
    sass = subprocess.check_output(["cuobjdump", "-sass", built_lib], text=True)

    def body(pattern):
        m = re.search(r"Function : \S*" + pattern + r".*?(?=Function :|\Z)", sass, re.S)
        assert m, pattern
        return m.group(0)
    atomic = re.compile(r"\b(RED|REDG|ATOM|ATOMG|ATOMS)\.")
    for t in ("f", "d"):
        for k in ("spmm_coo_sorted_kernelI" + t, "spmm_coo_fixup_kernelI" + t, "spmm_coo_scale_kernelI" + t):
            b = body(k)
            assert not atomic.search(b) and "STL" not in b and "LDL" not in b, k
        b = body("spmm_coo_atomic_kernelI" + t)
        assert atomic.search(b) and "STL" not in b
    b = body("spmm_coo_check_kernel")
    assert not atomic.search(b) and "STL" not in b
