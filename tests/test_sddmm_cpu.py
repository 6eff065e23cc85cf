"""CPU: the SDDMM additions to libb200spmv.so without a device -- symbols, the reference samples' goldens, the int64 reference
against scipy, the kernel's chunk walk at the edges built from b200sddmm_params, the routing table over real descriptors,
host-side argument rejection, and what the kernel compiles to."""
import ctypes as C
import os
import re
import subprocess
import sys
import textwrap

import numpy as np
import pytest

from oracle import exact as X
from oracle import sddmm_ref as R
from test_abi import declared_symbols, exported, kernel_sass

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REAL = "/usr/local/cuda/lib64/libcusparse.so.12"
NEW = ["cusparseSDDMM_bufferSize", "cusparseSDDMM_preprocess", "cusparseSDDMM", "b200sddmm_csr", "b200sddmm_csr_workspace_bytes",
       "b200sddmm_params", "b200sddmm_route"]


def test_header_declares_and_library_exports_the_sddmm_symbols(built_lib):
    names = declared_symbols()
    have = exported(built_lib)
    for n in NEW:
        assert n in names and n in have, n


def test_reference_goldens_of_both_samples():
    S = R.samples()
    s = S["sddmm_csr"]
    a = np.array(s["A"]).reshape(s["m"], s["k"])
    b = np.array(s["B"]).reshape(s["k"], s["n"])
    assert np.array_equal(R.reference(s["off"], s["col"], a, b, None, s["alpha"], s["beta"]), s["C_result"])
    s = S["sddmm_csr_batched"]
    for A, B, col, gold in zip(s["A"], s["B"], s["col"], s["C_result"]):
        a = np.array(A).reshape(s["m"], s["k"])
        b = np.array(B).reshape(s["k"], s["n"])
        assert np.array_equal(R.reference(s["off"], col, a, b, None, 1.0, 0.0), gold)


@pytest.mark.parametrize("kind", ["f32", "f64", "wide"])
@pytest.mark.parametrize("base", [0, 1])
def test_int64_reference_matches_scipy(kind, base):
    lens = [0, 3, 17, 0, 1, 40, 2]
    off, col = X.lens_to_structure(lens, 45, 1)
    off, col = off + base, col + base
    a, b, c0 = R.values(kind, len(lens), 45, 33, len(col), 2)
    R.check_exact(off, col, a, b, c0, -2.0, 0.5, R.MANTISSA[kind], base)
    sp = R.scipy_reference(off, col, a, b, base)
    assert np.array_equal(R.dots(off, col, a, b, base).astype(np.float64), sp.data) or np.array_equal(
        R.dots(off, col, a, b, base)[np.lexsort((col, R.rows_of(off, base)))].astype(np.float64), sp.data)
    got = R.reference(off, col, a, b, c0, -2.0, 0.5, base)
    assert np.array_equal(got, -2.0 * R.dots(off, col, a, b, base) + 0.5 * c0)


def test_wide_values_need_more_than_fp32():
    off, col = X.lens_to_structure([20, 30], 40, 3)
    a, b, _ = R.values("wide", 2, 40, 64, len(col), 4)
    assert R.dots(off, col, a, b, absolute=True).max() >= 1 << 24


def test_chunk_walk_computes_every_entry_once(built_lib):
    lib = C.CDLL(built_lib)
    P = R.params(lib)
    w = P["warp_chunk"]
    lens = []
    pos = 0
    for target in (w - 1, w, w + 1, 2 * w - 1, 2 * w + 1, 3 * w):
        if target > pos:
            lens.append(target - pos)
            pos = target
        lens.append(0)
    lens += [5 * w + 3, 0, 0, 1, w, 1, 0]
    off = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    true_rows = R.rows_of(off)
    ends = set(off[1:].tolist())
    assert {w - 1, w, w + 1, 2 * w - 1, 2 * w + 1} <= ends      # row ends at the chunk borders +- 1
    assert max(lens) > 4 * w                                       # one row longer than several chunks
    for itemsize in (4, 8):
        v = P["vec_bytes"] // itemsize
        for k in R.k_edges(P, itemsize):
            for vw in (1, v):
                visits, used = R.chunk_walk(off, int(off[-1]), k, vw, P)
                assert (visits == 1).all() and np.array_equal(used, true_rows), (k, vw)


def test_k_edges_cover_every_group_width(built_lib):
    P = R.params(C.CDLL(built_lib))
    for itemsize in (4, 8):
        v = P["vec_bytes"] // itemsize
        ks = R.k_edges(P, itemsize)
        for vw in (1, v):
            groups = {R.group(k, vw, P["max_group"]) for k in ks}
            assert groups == {1, 2, 4, 8, 16, 32}
        assert max(ks) > 2 * P["max_group"] * v                   # several passes of the widest group


ROUTE = textwrap.dedent("""
    import ctypes as C, sys
    real = C.CDLL(sys.argv[2], mode=C.RTLD_GLOBAL)
    shim = C.CDLL(sys.argv[1])
    I32, I64, F32, F64, F16, C32 = 2, 3, 0, 1, 2, 4
    ROW, COL = 2, 1
    NT, TR, CT = 0, 1, 2
    buf = (C.c_double * 4096)()
    off = (C.c_int * 5)(0, 1, 2, 3, 4)
    off64 = (C.c_int64 * 5)(0, 1, 2, 3, 4)

    def dn(r, c, vt=F32, order=ROW, batches=1, stride=0):
        d = C.c_void_p()
        assert real.cusparseCreateDnMat(C.byref(d), C.c_int64(r), C.c_int64(c), C.c_int64(c if order == ROW else r), buf, vt, order) == 0
        if batches > 1:
            assert real.cusparseDnMatSetStridedBatch(d, batches, C.c_int64(stride)) == 0
        return d

    def csr(vt=F32, idx=I32, batches=1, off_stride=0, cv_stride=4, lib=shim):
        d = C.c_void_p()
        o = off64 if idx == I64 else off
        assert lib.cusparseCreateCsr(C.byref(d), C.c_int64(4), C.c_int64(3), C.c_int64(4), o, buf, buf, idx, idx, 0, vt) == 0
        if batches > 1:
            assert lib.cusparseCsrSetStridedBatch(d, batches, C.c_int64(off_stride), C.c_int64(cv_stride)) == 0
        return d

    route = lambda a, b, c, opA=NT, opB=NT, ct=F32: shim.b200sddmm_route(a, b, c, opA, opB, ct)
    A, B, Cm = dn(4, 5), dn(5, 3), csr()
    if sys.argv[3] == "forward":
        assert route(A, B, Cm) == 0                                  # B200SPMV_FORWARD=1: everything to the closed library
        print("OK"); sys.exit(0)
    assert route(A, B, Cm) == 1
    for opA in (NT, TR):
        for opB in (NT, TR):
            for oa in (ROW, COL):
                for ob in (ROW, COL):
                    a = dn(4, 5, order=oa) if opA == NT else dn(5, 4, order=oa)
                    b = dn(5, 3, order=ob) if opB == NT else dn(3, 5, order=ob)
                    assert route(a, b, Cm, opA, opB) == 1, (opA, opB, oa, ob)
    # measured speed decides (DESIGN.md 3.13): fp64 and fp32 with K > 32 on a K-contiguous op(B) go to the closed library
    assert route(dn(4, 5, F64), dn(5, 3, F64), csr(F64), ct=F64) == 0
    assert route(dn(4, 32), dn(3, 32), Cm, opB=TR) == 1                        # fp32, K = 32, K-contiguous
    assert route(dn(4, 33), dn(3, 33), Cm, opB=TR) == 0                        # fp32, K = 33, K-contiguous
    assert route(dn(4, 64), dn(64, 3), Cm) == 1                                # fp32, K = 64, the sample's layout (B K x N row-major)
    assert route(dn(4, 64), dn(64, 3, order=COL), Cm) == 0                     # fp32, K = 64, column-major B: K-contiguous
    assert route(dn(4, 5), dn(6, 3), Cm) == 1                                  # a shape mismatch stays native: rejected by the call
    assert route(A, B, Cm, opA=CT) == 0 and route(A, B, Cm, opB=CT) == 0      # CONJUGATE_TRANSPOSE
    assert route(A, B, csr(idx=I64)) == 0                                      # 64-bit indices
    assert route(A, B, Cm, ct=F64) == 0                                        # compute type != value type
    assert route(dn(4, 5, F16), dn(5, 3, F16), csr(F16)) == 0                  # 16-bit
    assert route(dn(4, 5, C32), dn(5, 3, C32), csr(C32), ct=C32) == 0          # complex
    assert route(dn(4, 5, F64), B, Cm) == 0                                    # mixed types
    assert route(dn(4, 5, F64), dn(5, 3, F64), csr(F32), ct=F64) == 0
    # strided batches: C has N, A and B N or 1; shared offsets; outputs apart
    Cb = csr(batches=2, off_stride=0, cv_stride=4)
    assert route(dn(4, 5, batches=2, stride=20), dn(5, 3, batches=2, stride=15), Cb) == 2            # the batched sample's layout
    assert route(A, dn(5, 3, batches=2, stride=15), Cb) == 2                                         # A shared
    assert route(dn(4, 5, batches=2, stride=20), B, Cb) == 2                                         # B shared
    assert route(A, B, Cb) == 2
    assert route(A, B, csr(batches=2, off_stride=5, cv_stride=4)) == 2                              # per-matrix offsets
    assert route(dn(4, 5, batches=3, stride=20), B, Cb) == 0                                         # 3 of A for 2 of C
    assert route(A, dn(5, 3, batches=3, stride=15), Cb) == 0
    assert route(dn(4, 5, batches=2, stride=20), B, Cm) == 0                                         # a batch of A, one C
    Co = csr()                                                                                       # overlapping outputs: refused by the
    assert shim.cusparseCsrSetStridedBatch(Co, 2, C.c_int64(0), C.c_int64(3)) != 0                   # real library itself, and not recorded
    assert route(A, B, Co) == 1
    # recorded vs real batch count: set on the real descriptor behind the shim's back -> strides unknown -> forwarded
    Cr = csr()
    assert real.cusparseCsrSetStridedBatch(Cr, 2, C.c_int64(0), C.c_int64(4)) == 0
    assert route(A, B, Cr) == 0
    # a CSR descriptor the shim never saw: found through the real getters, one product
    assert route(A, B, csr(lib=real)) == 1
    assert route(None, B, Cm) == 0
    print("OK")
""")


@pytest.mark.parametrize("mode", ["default", "forward"])
def test_route_table_over_real_descriptors(built_lib, mode):
    if not os.path.exists(REAL):
        pytest.skip("no toolkit libcusparse here")
    env = {k: v for k, v in os.environ.items() if not k.startswith("B200SPMV_")}
    env["B200SPMV_CUSPARSE"] = REAL
    if mode == "forward":
        env["B200SPMV_FORWARD"] = "1"
    p = subprocess.run([sys.executable, "-c", ROUTE, built_lib, REAL, mode], capture_output=True, text=True, timeout=120, env=env)
    assert p.returncode == 0 and p.stdout.strip().endswith("OK"), p.stdout + p.stderr


def test_host_side_argument_rejection(built_lib):
    lib = C.CDLL(built_lib)
    one = C.c_float(1.0)
    dummy = (C.c_int * 8)()

    def call(dtype=0, m=4, n=3, k=5, nnz=4, off=dummy, col=dummy, val=dummy, base=0, alpha=C.byref(one), beta=C.byref(one), A=dummy,
             sai=5, sak=1, B=dummy, sbk=3, sbj=1, batch=1, os_=0, cv=0, as_=0, bs=0):
        return lib.b200sddmm_csr(None, dtype, C.c_int64(m), C.c_int64(n), C.c_int64(k), C.c_int64(nnz), off, col, val, base, alpha, beta,
                                 0, A, C.c_int64(sai), C.c_int64(sak), B, C.c_int64(sbk), C.c_int64(sbj), batch, C.c_int64(os_),
                                 C.c_int64(cv), C.c_int64(as_), C.c_int64(bs), None, C.c_size_t(0))
    assert call(dtype=2) == -1
    assert call(m=-1) == -1 and call(k=-1) == -1 and call(nnz=-1) == -1
    assert call(alpha=None) == -1 and call(beta=None) == -1
    assert call(base=2) == -1
    assert call(batch=0) == -1 and call(batch=65536) == -1
    assert call(batch=2, cv=3) == -1                                 # the batch's outputs would overlap
    assert call(sai=-1) == -1 and call(as_=-1) == -1
    assert call(off=None) == -1 and call(col=None) == -1 and call(val=None) == -1
    assert call(A=None) == -1 and call(B=None) == -1
    assert call(m=0, nnz=4) == -1
    assert call(m=1 << 31) == -1 and call(nnz=1 << 31) == -1
    assert call(nnz=0) == 0 and call(m=0, nnz=0) == 0              # nothing to do: no launch
    ws = lib.b200sddmm_csr_workspace_bytes
    ws.restype = C.c_size_t
    i64 = C.c_int64
    assert ws(0, i64(10), i64(20), i64(8), i64(8), i64(1), i64(1), i64(8), 1, i64(0), i64(0)) == 0          # both K-contiguous
    assert ws(0, i64(10), i64(20), i64(8), i64(8), i64(1), i64(20), i64(1), 1, i64(0), i64(0)) == 768        # B copied: 640 B -> 768
    assert ws(1, i64(10), i64(20), i64(8), i64(1), i64(10), i64(20), i64(1), 2, i64(80), i64(0)) == 1280 + 1280
    assert ws(0, i64(10), i64(20), i64(1), i64(1), i64(10), i64(20), i64(1), 1, i64(0), i64(0)) == 0         # K = 1: nothing to copy


def test_sass_of_the_sddmm_kernel(built_lib):
    """the K-contiguous instantiation loads A and B 128 bits per lane through the read-only path; no kernel spills to local memory;
    no tensor cores; no getenv in the source"""
    body = kernel_sass(built_lib, r"sddmm_csr_kernelIfLi4E")
    assert re.search(r"LDG\.E\.128\.CONSTANT", body)
    assert "SHFL.BFLY" in body and "HMMA" not in body
    for inst in ("sddmm_csr_kernelIfLi4E", "sddmm_csr_kernelIfLi1E", "sddmm_csr_kernelIdLi2E", "sddmm_csr_kernelIdLi1E"):
        assert "STL" not in kernel_sass(built_lib, inst), inst
    assert re.search(r"LDG\.E\.128\.CONSTANT", kernel_sass(built_lib, r"sddmm_csr_kernelIdLi2E"))
    assert "getenv(" not in open(os.path.join(ROOT, "cudalibrarysamples_b200", "csrc", "sddmm_csr.cu")).read()
