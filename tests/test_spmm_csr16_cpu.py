"""CPU: the half-precision CSR SpMM additions to libb200spmv.so without a device -- symbols, the int64 reference and its precondition,
the piece split's write-once property (with one very long row), the routing table over real descriptors, host-side argument
rejection, workspace bytes, path selection, params, and what the kernels compile to."""
import ctypes as C
import os
import re
import subprocess
import sys
import textwrap

import numpy as np
import pytest

from oracle import spmm_csr16_ref as R
from test_abi import declared_symbols, exported

REAL = "/usr/local/cuda/lib64/libcusparse.so.12"
NEW = ["b200spmm_csr16", "b200spmm_csr16_workspace_bytes", "b200spmm_csr16_path", "b200spmm_csr16_params", "b200spmm_csr16_route"]
F32, F64, F16, BF16 = 0, 1, 2, 14


def test_header_declares_and_library_exports_the_csr16_symbols(built_lib):
    names = declared_symbols()
    have = exported(built_lib)
    for n in NEW:
        assert n in names and n in have, n


@pytest.mark.parametrize("base", [0, 1])
def test_int64_reference_matches_scipy_and_checks_its_precondition(base):
    import scipy.sparse as sp
    lengths = [3, 0, 7, 1, 0, 12]
    off, col = R.pattern(lengths, 20, seed=1, base=base)
    val, b, c0 = R.values(6, 20, 9, len(col), seed=2)
    A = sp.csr_matrix((val, col - base, off - base), shape=(6, 20))
    assert np.array_equal(A @ b, R.products(off, col, val, b, base))
    got = R.reference_int(off, col, val, b, c0, -2.0, 0.5, "f16", base)
    assert np.array_equal(got, -2.0 * (A @ b) + 0.5 * c0)
    assert np.array_equal(R.reference_int(off, col, val, b, c0 * np.nan, 1.0, 0.0, "bf16", base), A @ b)
    big = np.full_like(b, 300)
    with pytest.raises(AssertionError):
        R.reference_int(off, col, np.abs(val), big, c0, 1.0, 0.0, "bf16", base)     # 300 does not fit the bf16 rule
    with pytest.raises(AssertionError):
        R.reference_int(off, col, val, b, c0, 3.0, 0.0, "f32", base)                 # alpha not a power of two


def lengths_with_a_long_row(P):
    return [0, 3, 40 * P + 17, 0, 1, P, P + 1, 2 * P - 1, 5, 0, 3 * P, 2, P - 1, 0]


PATTERNS = {
    "long": lambda P: lengths_with_a_long_row(P),
    "one-long-row": lambda P: [20000 + P // 3],
    "many-short": lambda P: [1, 2, 3, 0, 30, 31, 32, 33] * 40,
    "edges": lambda P: [P - 1, P, P + 1, 0, P + 1, P - 1, 2 * P, 2 * P + 1],
    "empty": lambda P: [0, 0, 0],
}


@pytest.mark.parametrize("name", sorted(PATTERNS))
def test_walk_writes_each_entry_once(built_lib, name):
    """both walks: every row written exactly once, every entry multiplied once, pieces at the row start + multiples of P; the split
    walk writes each carry slot once and the one fix-up of a long row reads exactly its pieces' slots in ascending piece order"""
    P = R.params(C.CDLL(built_lib))["piece"]
    lengths = PATTERNS[name](P)
    off = np.concatenate([[0], np.cumsum(lengths)]).astype(np.int64)
    m, nnz = len(lengths), int(off[-1])
    results = {}
    for split in (True, False):
        writes, reads, pieces = R.walk(off, P, split=split)
        rows = sorted(w[1] for w in writes if w[0] == "C")
        assert rows == list(range(m)), (split, rows)
        slots = [w[1] for w in writes if w[0] == "carry"]
        assert len(slots) == len(set(slots))
        assert all(s < 2 * (-(-nnz // P)) for s in slots)
        covered = sorted((p[1], p[2]) for p in pieces)
        assert [e for s, t in covered for e in range(s, t)] == list(range(nnz))
        for r, s, e, _ in pieces:
            assert off[r] <= s < e <= off[r + 1] and e - s <= P and (s - off[r]) % P == 0
        if split and nnz > P:
            for r in range(m):
                cnt = off[r + 1] - off[r]
                mine = [x for x in reads if x[2] == r]
                if cnt > P:
                    want = [R.slot(int(off[r]) + p * P, int(off[r]), P) for p in range(-(-cnt // P))]
                    assert [x[1] for x in mine] == want and set(want) <= set(slots)
                    assert len({x[3] for x in mine}) == 1                      # one fix-up warp per long row
                    assert [w for w in writes if w[0] == "C" and w[1] == r][0][2][0] == "fixup"
                else:
                    assert not mine
            assert sorted(x[1] for x in reads) == sorted(slots)                # every slot written is read once
        results[split] = sorted((p[0], p[1], p[2]) for p in pieces)
    assert results[True] == results[False]                  # the same pieces: the same summation order, the same bits


def test_walk_spreads_a_long_row_over_many_warps(built_lib):
    P = R.params(C.CDLL(built_lib))["piece"]
    off = np.concatenate([[0], np.cumsum(lengths_with_a_long_row(P))])
    writes, _, pieces = R.walk(off, P)
    writers = {p[3] for p in pieces if p[0] == 2}
    assert len(writers) == 41 and ("tile", 0) in writers                   # 41 pieces, 41 different warps


ROUTE = textwrap.dedent("""
    import ctypes as C, sys
    real = C.CDLL(sys.argv[2], mode=C.RTLD_GLOBAL)
    shim = C.CDLL(sys.argv[1])
    shim.b200spmm_csr16_route.argtypes = [C.c_void_p] * 3 + [C.c_int] * 4
    for f in ("b200spmm_coo_route", "b200spmm_bsr_route", "b200spmm_bell_route"):
        getattr(shim, f).argtypes = [C.c_void_p] * 3 + [C.c_int] * 4
    shim.b200spmm_batch_count.argtypes = [C.c_void_p] * 3
    I32, I64 = 2, 3
    F32, F64, F16, BF16, C32, I8 = 0, 1, 2, 14, 4, 3
    ROW, COL = 2, 1
    NT, TR, CT = 0, 1, 2
    DEFAULT, COO_ALG1, CSR_ALG1, CSR_ALG2, CSR_ALG3, BSR_ALG1 = 0, 1, 4, 6, 12, 14
    buf = (C.c_double * (1 << 20))()
    idx = (C.c_int * 4096)()

    def csr(rows, cols, nnz, vt=F16, it=I32, lib=shim, batch=1):
        d = C.c_void_p()
        assert lib.cusparseCreateCsr(C.byref(d), C.c_int64(rows), C.c_int64(cols), C.c_int64(nnz), idx, idx, buf, it, it, 0, vt) == 0
        if batch > 1:
            assert lib.cusparseCsrSetStridedBatch(d, batch, C.c_int64(0), C.c_int64(nnz)) == 0
        return d

    def dn(r, c, vt=F16, order=ROW, batches=1):
        d = C.c_void_p()
        assert real.cusparseCreateDnMat(C.byref(d), C.c_int64(r), C.c_int64(c), C.c_int64(c if order == ROW else r), buf, vt, order) == 0
        if batches > 1:
            assert real.cusparseDnMatSetStridedBatch(d, batches, C.c_int64(r * c)) == 0
        return d

    route = lambda a, b, c, opA=NT, opB=NT, ct=F32, alg=DEFAULT: shim.b200spmm_csr16_route(a, b, c, opA, opB, ct, alg)
    native = eval(sys.argv[4])               # the measured classes: (type, c type, n, m, nnz, order) -> native
    forward = sys.argv[3] == "forward"
    for vt, cvt in ((F16, F16), (F16, F32), (BF16, BF16), (BF16, F32)):
        for n in (8, 32, 64, 128, 256, 512):
            for m, per in ((1 << 16, 16), (1 << 20, 4), (1 << 20, 16), (2 << 20, 32)):
                for order in (ROW, COL):
                    a = csr(m, m, m * per, vt)
                    r = route(a, dn(m, n, vt, order), dn(m, n, cvt, order))
                    want = 0 if forward else int(native(vt, cvt, n, m, m * per, order))
                    assert r == want, (vt, cvt, n, m, per, order, r)
                    assert route(a, dn(m, n, vt, ROW), dn(m, n, cvt, COL)) == 0                 # mixed orders: not measured
    if forward:
        print("OK"); sys.exit(0)
    # a natively routed class, if the table has one, to check every forwarded variant against
    cls = [(vt, cvt, n, m, per, order) for vt, cvt in ((F16, F16), (F16, F32), (BF16, BF16), (BF16, F32)) for n in (32, 64, 128, 256)
           for m, per in ((1 << 20, 16), (2 << 20, 32)) for order in (ROW, COL) if native(vt, cvt, n, m, m * per, order)]
    vt, cvt, n, m, per, order = cls[0] if cls else (F16, F16, 128, 1 << 20, 16, ROW)
    A = lambda **kw: csr(m, m, m * per, **{"vt": vt, **kw})
    B, Cm = dn(m, n, vt, order), dn(m, n, cvt, order)
    ok = 1 if cls else 0
    assert route(A(), B, Cm) == ok
    for alg in (CSR_ALG1, CSR_ALG2, CSR_ALG3):
        assert route(A(), B, Cm, alg=alg) == ok, alg
    for alg in (COO_ALG1, BSR_ALG1):                                            # other algorithms: forwarded
        assert route(A(), B, Cm, alg=alg) == 0, alg
    assert route(A(), B, Cm, opA=TR) == 0 and route(A(), B, Cm, opA=CT) == 0    # opA = T / C: forwarded
    assert route(A(), B, Cm, opB=CT) == 0
    assert route(A(), dn(n, m, vt, COL if order == ROW else ROW), Cm, opB=TR) == 0   # opB = T: not measured
    assert route(A(it=I64), B, Cm) == 0                                         # 64-bit indices
    assert route(A(), B, Cm, ct=F16) == 0                                       # 16-bit compute
    assert route(A(), dn(m, n, F32, order), dn(m, n, F32, order)) == 0          # mixed A / B types
    other = BF16 if vt == F16 else F16
    assert route(A(), B, dn(m, n, other, order)) == 0                           # C of the other 16-bit type
    assert route(A(vt=I8), dn(m, n, I8, order), dn(m, n, F32, order), ct=F32) == 0   # int8
    assert route(A(batch=4), dn(m, n, vt, order, 4), dn(m, n, cvt, order, 4)) == 0  # strided batches
    assert route(A(), B, dn(m, n, cvt, order, 4)) == 0
    assert route(A(lib=real), B, Cm) == ok                                      # created behind the shim's back: the real getter
    assert route(A(), dn(m + 1, n, vt, order), Cm) == ok                        # a shape mismatch stays: the call rejects it
    assert route(None, B, Cm) == 0 and route(A(), None, Cm) == 0
    # fp32 / fp64 CSR and the other formats are not this route's; the batch count of a 16-bit CSR A is as before
    assert route(csr(m, m, m * per, F32), dn(m, n, F32, order), dn(m, n, F32, order)) == 0
    assert shim.b200spmm_batch_count(A(), B, Cm) == 1
    assert shim.b200spmm_batch_count(A(batch=4), dn(m, n, vt, order, 4), dn(m, n, cvt, order, 4)) == 0
    print("OK")
""")


def native_table():
    """the route's table (DESIGN.md 3.18), as the predicate the script evaluates: (type, c type, n, m, nnz, order) -> native"""
    from scripts.spmm_csr16_bench import NATIVE
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


def test_host_side_argument_rejection(built_lib):
    lib = C.CDLL(built_lib)
    i64, vp = C.c_int64, C.c_void_p
    lib.b200spmm_csr16.argtypes = [vp, C.c_int, C.c_int, i64, i64, i64, i64, vp, vp, vp, C.c_int32, vp, vp, C.c_int, vp, i64, i64, vp,
                                   i64, C.c_int, vp, C.c_size_t]
    one = C.c_float(1.0)
    dummy = (C.c_int * 64)()
    p = C.addressof(dummy)
    o = C.addressof(one)

    def call(at=F16, ct=F16, m=32, k=32, n=8, nnz=2, off=p, col=p, val=p, base=0, alpha=o, beta=o, B=p, sbk=8, sbj=1, Cm=p, ldc=8, crow=1):
        return lib.b200spmm_csr16(None, at, ct, m, k, n, nnz, off, col, val, base, alpha, beta, 0, B, sbk, sbj, Cm, ldc, crow, None, 0)
    assert call(at=F32, ct=F32) == -1 and call(at=F64, ct=F64) == -1 and call(at=3) == -1         # fp32 / fp64 are spmm_csr.cu's
    assert call(ct=BF16) == -1 and call(at=BF16, ct=F16) == -1 and call(ct=F64) == -1
    assert call(m=-1) == -1 and call(k=-1) == -1 and call(n=-1) == -1 and call(nnz=-1) == -1
    assert call(nnz=32 * 32 + 1) == -1                                                # more entries than the matrix holds
    assert call(base=2) == -1 and call(alpha=None) == -1 and call(beta=None) == -1
    assert call(sbk=-1) == -1 and call(sbj=-1) == -1
    assert call(ldc=7) == -1 and call(crow=0, ldc=31) == -1                          # ldc below the tight one
    assert call(off=None) == -1 and call(col=None) == -1 and call(val=None) == -1 and call(B=None) == -1 and call(Cm=None) == -1
    assert call(m=0, nnz=0) == 0 and call(n=0) == 0                                  # nothing to do: no launch
    assert call(m=1 << 32, k=1 << 32) == -1 and call(n=1 << 22) == -1


def test_workspace_bytes(built_lib):
    """the row-major copy of a K-contiguous op(B) (256-byte rounded), then two carry slots of n fp32 partial sums per chunk of P
    entries"""
    lib = C.CDLL(built_lib)
    lib.b200spmm_csr16_workspace_bytes.argtypes = [C.c_int64] * 5
    lib.b200spmm_csr16_workspace_bytes.restype = C.c_size_t
    P = R.params(lib)["piece"]
    ws = lib.b200spmm_csr16_workspace_bytes
    for k, n, nnz in ((1 << 20, 128, 16 << 20), (1000, 7, 1), (5, 256, 3 * P + 1)):
        carry = 2 * (-(-nnz // P)) * n * 4
        assert ws(k, n, nnz, n, 1) == carry                                          # N-contiguous op(B): no copy
        assert ws(k, n, nnz, 1, k) == carry + (-(-(k * n * 2) // 256)) * 256          # K-contiguous: the copy too
    assert ws(100, 1, 10, 1, 1) == 2 * 4                                             # n = 1: nothing to copy
    assert ws(100, 64, 0, 1, 100) == 0 and ws(100, 0, 10, 64, 1) == 0


def test_path_selection(built_lib):
    lib = C.CDLL(built_lib)
    lib.b200spmm_csr16_path.argtypes = [C.c_int64, C.c_void_p, C.c_int64, C.c_int64]
    path = lambda n=128, B=4096, sbk=128, sbj=1: lib.b200spmm_csr16_path(n, B, sbk, sbj)  # noqa: E731
    assert path() == 4 and path(n=64, sbk=64) == 2 and path(n=256, sbk=256) == 8 and path(n=129, sbk=136) == 8
    assert path(n=32, sbk=32) == 1 and path(n=1, sbk=1) == 1                          # one column per lane
    assert path(B=4098) == 1 and path(n=256, B=4104, sbk=256) == 1                    # misaligned views
    assert path(sbk=130) == 1 and path(n=64, sbk=65) == 1                             # a leading dimension not a multiple of V
    assert path(sbk=1, sbj=4096) == 1                                                 # K-contiguous in place: scalar
    assert path(n=0) == 0 and path(sbk=-1) == 0


def test_params(built_lib):
    P = R.params(C.CDLL(built_lib))
    assert P["piece"] >= 64 and P["lane_entries"] == 32 and P["tile_rows"] % P["warps"] == 0 and P["max_cols_per_lane"] == 8


def test_sass_of_the_csr16_kernels(built_lib):
    """fp32 accumulation on FFMA, no tensor instruction, no local memory; the vector paths gather with one 128 / 64 / 32-bit load"""
    sass = subprocess.check_output(["cuobjdump", "-sass", built_lib], text=True)
    bodies = {}
    for m in re.finditer(r"Function : (\S*spmm_csr16_\S*)(.*?)(?=Function :|\Z)", sass, re.S):
        bodies[m.group(1)] = m.group(2)
    main = [k for k in bodies if "spmm_csr16_kernel" in k]
    assert len(main) == 2 * 7 * 2 and len([k for k in bodies if "fixup" in k]) == 2, sorted(bodies)
    for name, body in bodies.items():
        assert "HMMA" not in body and "STL" not in body and "LDL" not in body, name
        assert "FFMA" in body or "fixup" in name, name
    for t in ("6__half", "13__nv_bfloat16"):
        for v, width in ((8, "128"), (4, "64")):
            body = bodies[f"_ZN4b20017spmm_csr16_kernelI{t}Li{v}ELi{v}ELb1EEEvNS_13SpmmCsr16ArgsENS_7ScalarsIfEE"]
            assert re.search(rf"LDG\.E\.{width}\.CONSTANT", body), (t, v)
