"""CPU: the shim's descriptor side (no device needed -- the real library's descriptor calls are host-only): descriptors created
through the shim's cusparseCreateCsr stay real descriptors, cusparseCsrSetStridedBatch reaches the real library AND the side
table, and the strided-batch decision of cusparseSpMM (b200spmm_batch_count) follows B200SPMV_GENERIC.  Runs in a subprocess:
the shim picks its real libcusparse once per process (B200SPMV_CUSPARSE)."""
import os
import subprocess
import sys
import textwrap

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REAL = "/usr/local/cuda/lib64/libcusparse.so.12"

SCRIPT = textwrap.dedent("""
    import ctypes as C, os, sys
    sys.path.insert(0, os.path.dirname(os.path.dirname(sys.argv[1])))     # the repository: argv[1] is its built library
    from cudalibrarysamples_b200.lib import load
    real = C.CDLL(sys.argv[2], mode=C.RTLD_GLOBAL)
    shim = load(sys.argv[1])
    I32, F32, COL = 2, 0, 1
    off = (C.c_int * 5)(0, 3, 4, 7, 9)
    col = (C.c_int * 18)()
    val = (C.c_float * 18)()
    B = (C.c_float * 24)()
    Cm = (C.c_float * 24)()

    def csr(lib):
        d = C.c_void_p()
        assert lib.cusparseCreateCsr(C.byref(d), C.c_int64(4), C.c_int64(4), C.c_int64(9), off, col, val, I32, I32, 0, F32) == 0
        return d

    def dn(batches, stride):
        d = C.c_void_p()
        assert real.cusparseCreateDnMat(C.byref(d), C.c_int64(4), C.c_int64(3), C.c_int64(4), B, F32, COL) == 0
        if batches > 1:
            assert real.cusparseDnMatSetStridedBatch(d, batches, C.c_int64(stride)) == 0
        return d

    def count(a, b, c):
        return shim.b200spmm_batch_count(a, b, c)

    def mode(m):
        assert shim.b200spmv_set_option(b"B200SPMV_GENERIC", m) == 0

    A = csr(shim)
    n = C.c_int(-1)
    assert real.cusparseSpMatGetStridedBatch(A, C.byref(n)) == 0 and n.value == 1     # a real descriptor, not batched
    for m in (b"off", b"csr", b"all"):
        mode(m)
        assert count(A, dn(1, 0), dn(1, 0)) == 1                                       # the ordinary product, whatever the switch says
    # spmm_csr_batched_example.c:140-148: shared offsets, per-batch columns / values, B and C strided
    assert shim.cusparseCsrSetStridedBatch(A, 2, C.c_int64(0), C.c_int64(9)) == 0
    assert real.cusparseSpMatGetStridedBatch(A, C.byref(n)) == 0 and n.value == 2     # the real descriptor saw it too
    mode(b"csr")
    assert count(A, dn(2, 12), dn(2, 12)) == 0                                         # default: batches go to the closed library
    mode(b"all")
    assert count(A, dn(2, 12), dn(2, 12)) == 2
    assert count(A, dn(1, 0), dn(2, 12)) == 2                                          # B shared by the batch
    assert count(A, dn(2, 12), dn(3, 12)) == 0                                         # 2 matrices, 3 outputs
    assert count(A, dn(3, 12), dn(2, 12)) == 0
    d = C.c_void_p()                                                                   # overlapping outputs: the real library refuses the stride itself
    assert real.cusparseCreateDnMat(C.byref(d), C.c_int64(4), C.c_int64(3), C.c_int64(4), B, F32, COL) == 0
    assert real.cusparseDnMatSetStridedBatch(d, 2, C.c_int64(6)) != 0
    A1 = csr(shim)                                                                     # one matrix, batched right-hand sides (":141-142 broadcast")
    assert count(A1, dn(2, 12), dn(2, 12)) == 2
    # a batch set behind the shim's back (the real symbol called directly): strides unknown -> not ours
    A2 = csr(shim)
    assert real.cusparseCsrSetStridedBatch(A2, 2, C.c_int64(0), C.c_int64(9)) == 0
    assert count(A2, dn(2, 12), dn(2, 12)) == 0
    # a descriptor the shim never saw: found through the real getters, ordinary product only
    A3 = csr(real)
    assert count(A3, dn(1, 0), dn(1, 0)) == 1
    # every descriptor kind the samples create goes through the shim and stays a REAL descriptor: the real getters see what
    # the shim was given (spmv_coo_example.c:86-89, spmv_sell_example.c:103-107, spmv_csr_example.c:93-95), set-pointer calls reach both sides
    fmt = C.c_int(-1)
    coo = C.c_void_p()
    assert shim.cusparseCreateCoo(C.byref(coo), C.c_int64(4), C.c_int64(4), C.c_int64(9), col, col, val, I32, 0, F32) == 0
    assert real.cusparseSpMatGetFormat(coo, C.byref(fmt)) == 0 and fmt.value == 3
    sell = C.c_void_p()
    assert shim.cusparseCreateSlicedEll(C.byref(sell), C.c_int64(4), C.c_int64(4), C.c_int64(9), C.c_int64(12), C.c_int64(2), off, col, val,
                                        I32, I32, 0, F32) == 0
    assert real.cusparseSpMatGetFormat(sell, C.byref(fmt)) == 0 and fmt.value == 7
    vec = C.c_void_p()
    assert shim.cusparseCreateDnVec(C.byref(vec), C.c_int64(4), B, F32) == 0
    size, vals, vt = C.c_int64(), C.c_void_p(), C.c_int()
    assert real.cusparseDnVecGet(vec, C.byref(size), C.byref(vals), C.byref(vt)) == 0 and size.value == 4 and vals.value == C.addressof(B)
    assert shim.cusparseDnVecSetValues(vec, Cm) == 0
    assert real.cusparseDnVecGetValues(vec, C.byref(vals)) == 0 and vals.value == C.addressof(Cm)
    off2 = (C.c_int * 5)(0, 1, 2, 3, 4)
    assert shim.cusparseCsrSetPointers(A1, off2, col, val) == 0
    r, c_, z, po, pc, pv = C.c_int64(), C.c_int64(), C.c_int64(), C.c_void_p(), C.c_void_p(), C.c_void_p()
    ot, ct, ib, vt2 = C.c_int(), C.c_int(), C.c_int(), C.c_int()
    assert real.cusparseCsrGet(A1, C.byref(r), C.byref(c_), C.byref(z), C.byref(po), C.byref(pc), C.byref(pv), C.byref(ot), C.byref(ct),
                               C.byref(ib), C.byref(vt2)) == 0 and po.value == C.addressof(off2) and (r.value, c_.value, z.value) == (4, 4, 9)
    assert shim.cusparseDestroyDnVec(vec) == 0
    for d in (coo, sell):
        assert shim.cusparseDestroySpMat(d) == 0
    # what cusparseSpMV would do with descriptors like these (b200spmv_route), under the default switch
    mode(b"csr")
    assert shim.b200spmv_route(1, 0, 0, I32, I32, F32, F32, F32, F32, C.c_int64(4), C.c_int64(4), C.c_int64(9)) == 1
    for d in (A, A1, A2):
        assert shim.cusparseDestroySpMat(d) == 0
    assert real.cusparseDestroySpMat(A3) == 0
    # cusparseCreateX and cusparseCreateConstX through the shim, for every kind it records: the real getters see the same values, and
    # the route exports give both the same (native) answer -- a BSR descriptor the shim did not record would be forwarded
    I64, VP, INT = C.c_int64, C.c_void_p, C.c_int
    F16, ROW, NT, TR = 2, 2, 0, 1
    big = (C.c_double * (1 << 20))()
    at = C.addressof

    def both(kind, *args):
        made = []
        for f in ("cusparseCreate" + kind, "cusparseCreateConst" + kind):
            d = C.c_void_p()
            assert getattr(shim, f)(C.byref(d), *args) == 0, f
            made.append(d)
        return made

    def get(fn, d, *types):
        out = [t() for t in types]
        assert getattr(real, fn)(d, *[C.byref(o) for o in out]) == 0, fn
        return [o.value for o in out]

    def spmat(d):                                          # what every sparse descriptor answers (no Sliced-ELL / BSR getter exists)
        return (get("cusparseSpMatGetFormat", d, INT) + get("cusparseSpMatGetSize", d, I64, I64, I64) +
                get("cusparseSpMatGetIndexBase", d, INT) + get("cusparseConstSpMatGetValues", d, VP))

    def dnm(r, c_, vt, order):
        d = C.c_void_p()
        assert real.cusparseCreateDnMat(C.byref(d), C.c_int64(r), C.c_int64(c_), C.c_int64(c_ if order == ROW else r), big, vt, order) == 0
        return d

    made = []
    pair = both("Csr", C.c_int64(4), C.c_int64(3), C.c_int64(4), off, col, val, I32, I32, 1, F32)
    for d in pair:
        csr_seen = get("cusparseConstCsrGet", d, I64, I64, I64, VP, VP, VP, INT, INT, INT, INT)
        assert csr_seen == [4, 3, 4, at(off), at(col), at(val), I32, I32, 1, F32]
        assert shim.b200sddmm_route(dnm(4, 5, F32, ROW), dnm(5, 3, F32, ROW), d, NT, NT, F32) == 1
    made += pair
    M = 1 << 16
    pair = both("Coo", C.c_int64(M), C.c_int64(48), C.c_int64(16 * M), off, col, val, I32, 0, F32)
    for d in pair:
        assert get("cusparseConstCooGet", d, I64, I64, I64, VP, VP, VP, INT, INT, INT) == [M, 48, 16 * M, at(off), at(col), at(val), I32, 0, F32]
        assert shim.b200spmm_coo_route(d, dnm(48, 32, F32, COL), dnm(M, 32, F32, COL), NT, NT, F32, 0) == 1
    made += pair
    pair = both("SlicedEll", C.c_int64(4), C.c_int64(4), C.c_int64(9), C.c_int64(12), C.c_int64(2), off, col, val, I32, I32, 0, F32)
    assert spmat(pair[0]) == spmat(pair[1]) == [7, 4, 4, 9, 0, at(val)]
    made += pair
    pair = both("Bsr", C.c_int64(256), C.c_int64(256), C.c_int64(64), C.c_int64(16), C.c_int64(16), off, col, big, I32, I32, 0, F16, ROW)
    assert spmat(pair[0]) == spmat(pair[1]) and spmat(pair[0])[0] == 6 and spmat(pair[0])[-1] == at(big)
    for d in pair:
        assert shim.b200sddmm_bsr_route(dnm(4096, 64, F16, ROW), dnm(4096, 64, F16, ROW), d, NT, TR, F32) == 1
    made += pair
    for d in made:
        assert shim.cusparseDestroySpMat(d) == 0
    for d in both("DnVec", C.c_int64(24), B, F32):
        assert get("cusparseConstDnVecGet", d, I64, VP, INT) == [24, at(B), F32]
        assert shim.cusparseDestroyDnVec(d) == 0
    print("OK")
""")


def test_descriptor_side_table_and_batch_decision(built_lib):
    import pytest
    if not os.path.exists(REAL):
        pytest.skip("no toolkit libcusparse here")
    env = {k: v for k, v in os.environ.items() if not k.startswith("B200SPMV_")}
    env["B200SPMV_CUSPARSE"] = REAL
    p = subprocess.run([sys.executable, "-c", SCRIPT, built_lib, REAL], capture_output=True, text=True, timeout=120, env=env)
    assert p.returncode == 0 and p.stdout.strip().endswith("OK"), p.stdout + p.stderr
