"""CPU: the BSR SpMM additions to libb200spmv.so without a device -- symbols, the int64 reference against scipy, the work split's
write-once property on the GPU tests' patterns, the routing table over real descriptors, host-side argument rejection, path
selection, params, and what the kernels compile to."""
import ctypes as C
import os
import re
import subprocess
import sys
import textwrap

import numpy as np
import pytest

from cudalibrarysamples_b200.lib import load
from oracle import spmm_bsr_ref as R
from test_abi import declared_symbols, exported

REAL = "/usr/local/cuda/lib64/libcusparse.so.12"
NEW = ["b200spmm_bsr", "b200spmm_bsr_workspace_bytes", "b200spmm_bsr_path", "b200spmm_bsr_params", "b200spmm_bsr_route"]
F32, F64, F16, BF16 = 0, 1, 2, 14


def test_header_declares_and_library_exports_the_bsr_spmm_symbols(built_lib):
    names = declared_symbols()
    have = exported(built_lib)
    for n in NEW:
        assert n in names and n in have, n


@pytest.mark.parametrize("bs", [1, 2, 3, 16, 64, 128])
@pytest.mark.parametrize("base", [0, 1])
@pytest.mark.parametrize("order", ["row", "col"])
def test_int64_reference_matches_scipy(bs, base, order):
    nbr, nbc = (5, 4) if bs <= 16 else (3, 2)
    off, col = R.pattern(nbr, nbc, [2, 0, 1, 4, 3], seed=bs, base=base)
    val, b, c0 = R.values(nbr * bs, nbc * bs, 7, len(col), bs, seed=3)
    A = R.to_scipy(nbr * bs, nbc * bs, bs, off, col, val, base, order)
    assert np.array_equal(A @ b, R.products(nbr * bs, nbc * bs, bs, off, col, val, b, base, order))
    got = R.reference(nbr * bs, nbc * bs, bs, off, col, val, b, c0, -2.0, 0.5, base, order)
    assert np.array_equal(got, -2.0 * (A @ b) + 0.5 * c0)
    assert np.array_equal(R.reference(nbr * bs, nbc * bs, bs, off, col, val, b, c0 * np.nan, 1.0, 0.0, base, order), A @ b)


def global_pattern(nb, seed=0):
    """the GPU tests' window-plus-global pattern: +-1 block columns, global block-row 1 and block column 0, one empty block-row"""
    mask = np.zeros((nb, nb), bool)
    for d in (-1, 0, 1):
        i = np.arange(max(0, -d), min(nb, nb - d))
        mask[i, i + d] = True
    mask[1, :] = True
    mask[:, 0] = True
    mask[nb - 2, :] = False
    off = np.concatenate([[0], np.cumsum(mask.sum(1))])
    return off, np.nonzero(mask)[1]


PATTERNS = {
    "global": lambda: global_pattern(40),
    "global-small": lambda: global_pattern(6),
    "uneven": lambda: R.pattern(9, 12, [0, 1, 12, 0, 3, 1, 0, 7], seed=2),
    "empty-ends": lambda: R.pattern(7, 5, [0, 2, 5, 0, 1, 0, 0], seed=4),
    "one-row": lambda: R.pattern(1, 30, [30], seed=5),
    "all-empty": lambda: (np.zeros(5, np.int64), np.zeros(0, np.int64)),
}


@pytest.mark.parametrize("name", sorted(PATTERNS))
def test_walk_writes_each_entry_once(built_lib, name):
    """both walks: every block-row written exactly once, every stored block multiplied exactly once in its row's piece order, carry
    slots written once and read in ascending piece order by the one fix-up that writes their row"""
    P = R.params(load(built_lib))
    off, col = PATTERNS[name]()
    bnnz = len(col)
    brows = len(off) - 1
    results = {}
    for split in (True, False):
        ch, writes, pieces = R.walk(off, bnnz, P, 16, 64, split=split)
        rows = [w[1] for w in writes if w[0] == "C"]
        assert sorted(rows) == list(range(brows)), (split, rows)
        slots = [w[1] for w in writes if w[0] == "carry"]
        assert len(slots) == len(set(slots))
        covered = sorted((p[2], p[3]) for p in pieces)
        assert [b for s, e in covered for b in range(s, e)] == list(range(bnnz))
        for _, r, s, e in pieces:
            assert off[r] <= s < e <= off[r + 1] and e - s <= ch and ((s - off[r]) % ch == 0)
        if split:
            for r in range(brows):
                cnt = off[r + 1] - off[r]
                if cnt > ch:
                    want = R.fixup_slots(off, r, ch)
                    assert len(want) == -(-cnt // ch) and set(want) <= set(slots) and want == sorted(want)
            assert all(s < 2 * (-(-bnnz // ch)) for s in slots)
        results[split] = sorted((p[1], p[2], p[3]) for p in pieces)
    assert results[True] == results[False]                  # the same pieces: the same summation order, the same bits


def test_walk_splits_a_global_row():
    P = dict(chunk_min=2, chunk_factor=2, target_ctas=1024)
    off, col = global_pattern(40)
    ch, writes, pieces = R.walk(off, len(col), P, 64, 128)
    assert off[2] - off[1] == 40 and ch < 40
    writers = {w[2] for w in writes if w[0] == "carry"}
    assert len(writers) >= 2                                  # the global block-row is spread over several CTAs


ROUTE = textwrap.dedent("""
    import ctypes as C, os, sys
    sys.path.insert(0, os.path.dirname(os.path.dirname(sys.argv[1])))     # the repository: argv[1] is its built library
    from cudalibrarysamples_b200.lib import load
    real = C.CDLL(sys.argv[2], mode=C.RTLD_GLOBAL)
    shim = load(sys.argv[1])
    I32, I64 = 2, 3
    F32, F64, F16, BF16, C32 = 0, 1, 2, 14, 4
    ROW, COL = 2, 1
    NT, TR, CT = 0, 1, 2
    DEFAULT, COO_ALG1, CSR_ALG2, BELL_ALG1, BSR_ALG1 = 0, 1, 6, 13, 14
    buf = (C.c_double * (1 << 20))()
    idx = (C.c_int * 4096)()

    def bsr(brows=64, bcols=64, bnnz=64, rbs=16, cbs=16, vt=F32, it=I32, order=ROW, lib=shim, batch=1, strides=(0, 0, 64 * 256)):
        d = C.c_void_p()
        assert lib.cusparseCreateBsr(C.byref(d), C.c_int64(brows), C.c_int64(bcols), C.c_int64(bnnz), C.c_int64(rbs), C.c_int64(cbs), idx,
                                     idx, buf, it, it, 0, vt, order) == 0
        if batch > 1:
            assert lib.cusparseBsrSetStridedBatch(d, batch, *[C.c_int64(s) for s in strides]) == 0
        return d

    def dn(r, c, vt=F32, order=ROW, batches=1):
        d = C.c_void_p()
        assert real.cusparseCreateDnMat(C.byref(d), C.c_int64(r), C.c_int64(c), C.c_int64(c if order == ROW else r), buf, vt, order) == 0
        if batches > 1:
            assert real.cusparseDnMatSetStridedBatch(d, batches, C.c_int64(r * c)) == 0
        return d

    route = lambda a, b, c, opA=NT, opB=NT, ct=F32, alg=DEFAULT: shim.b200spmm_bsr_route(a, b, c, opA, opB, ct, alg)
    native = eval(sys.argv[4])               # the measured classes: (type, c type, bs, n, m, order) -> native
    forward = sys.argv[3] == "forward"
    TYPES = ((F16, F16), (F16, F32), (BF16, BF16), (BF16, F32), (F32, F32), (F64, F64))
    for vt, cvt in TYPES:
        ct = F64 if vt == F64 else F32
        for bs in (2, 4, 8, 16, 32, 64, 128):
            for n in (8, 64, 128, 256):
                for m in (1024, 4096, 16384):
                    for order in (ROW, COL):
                        nb = m // bs
                        a = bsr(brows=nb, bcols=nb, bnnz=min(64, nb), rbs=bs, cbs=bs, vt=vt)
                        r = route(a, dn(m, n, vt, order), dn(m, n, cvt, order), NT, NT, ct)
                        want = 0 if forward else int(native(vt, cvt, bs, n, m, order))
                        assert r == want, (vt, cvt, bs, n, m, order, r)
    if forward:
        print("OK"); sys.exit(0)
    A = lambda **kw: bsr(brows=64, bcols=64, rbs=64, cbs=64, vt=F16, **kw)
    V, O = dn(4096, 64, F16), dn(4096, 64, F16)
    assert route(A(), V, O) == 1
    assert route(A(), V, O, alg=BSR_ALG1) == 1
    for alg in (COO_ALG1, CSR_ALG2, BELL_ALG1):                                              # other algorithms: forwarded
        assert route(A(), V, O, alg=alg) == 0, alg
    assert route(A(), V, O, opA=TR) == 0 and route(A(), V, O, opA=CT) == 0                   # opA = T / C: forwarded
    assert route(A(), dn(64, 4096, F16), O, opB=CT) == 0
    assert route(A(it=I64), V, O) == 0                                                         # 64-bit indices
    assert route(A(), V, O, ct=F16) == 0                                                       # 16-bit compute
    assert route(bsr(brows=64, bcols=64, rbs=64, cbs=64, vt=C32), dn(4096, 64, C32), dn(4096, 64, C32), ct=C32) == 0   # complex
    assert route(A(), dn(4096, 64, F32), dn(4096, 64, F32)) == 0                               # mixed A / B types
    assert route(A(order=COL), V, O) == 0                                                      # column-major blocks: not measured
    assert route(A(lib=real), V, O) == 0                                                       # created behind the shim's back
    assert route(A(), dn(4096, 48, F16), O) == 1                                               # a shape mismatch stays: the call rejects it
    assert route(None, V, O) == 0 and route(A(), None, O) == 0
    H = 16
    heads = lambda strides: A(batch=H, strides=strides)
    assert route(heads((0, 0, 64 * 4096)), dn(4096, 64, F16, batches=H), dn(4096, 64, F16, batches=H)) == H
    assert route(heads((0, 0, 64 * 4096)), V, dn(4096, 64, F16, batches=H)) == 0              # B shared by the batch
    assert route(heads((65, 64, 64 * 4096)), dn(4096, 64, F16, batches=H), dn(4096, 64, F16, batches=H)) == 0   # a pattern per head
    small = lambda bs, h: bsr(brows=4096 // bs, bcols=4096 // bs, rbs=bs, cbs=bs, vt=F16, batch=h, strides=(0, 0, 64 * bs * bs))
    assert route(small(16, 16), dn(4096, 64, F16, batches=16), dn(4096, 64, F16, batches=16)) == 16          # 16 heads at bs 16: measured
    assert route(small(16, 4), dn(4096, 64, F16, batches=4), dn(4096, 64, F16, batches=4)) == 0              # 4 heads: not measured
    assert route(small(32, 16), dn(4096, 64, F16, batches=16), dn(4096, 64, F16, batches=16)) == 0           # bs 32 heads: not measured
    # the SpMM batch count and the other routes still see a BSR A as before
    assert shim.b200spmm_batch_count(A(), V, O) == 0
    print("OK")
""")


def native_table():
    """the route's table (DESIGN.md 3.17), as the predicate the script evaluates: (type, c type, bs, n, m, order) -> native"""
    from scripts.spmm_bsr_bench import NATIVE
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
    lib = load(built_lib)
    one = C.c_float(1.0)
    dummy = (C.c_int * 64)()
    p = C.addressof(dummy)
    o = C.addressof(one)

    def call(at=F32, ct=F32, m=32, k=32, n=8, bs=16, bnnz=2, off=p, col=p, val=p, base=0, alpha=o, beta=o, B=p, sbk=8, sbj=1, Cm=p,
             ldc=8, crow=1, batch=1, st=(0, 0, 0, 0, 0)):
        return lib.b200spmm_bsr(None, at, ct, m, k, n, bs, bnnz, off, col, val, base, 1, alpha, beta, 0, B, sbk, sbj, Cm, ldc, crow, batch,
                                *st, None, 0)
    assert call(at=3) == -1 and call(ct=F64) == -1 and call(at=F16, ct=BF16) == -1 and call(at=F64, ct=F32) == -1
    assert call(m=-1) == -1 and call(k=-1) == -1 and call(bs=0) == -1 and call(bnnz=-1) == -1
    assert call(m=24) == -1 and call(k=24) == -1                                     # not multiples of bs
    assert call(bnnz=5) == -1                                                        # more blocks than the matrix holds
    assert call(base=2) == -1 and call(alpha=None) == -1 and call(beta=None) == -1
    assert call(sbk=-1) == -1 and call(batch=0) == -1 and call(batch=65536) == -1
    assert call(ldc=7) == -1 and call(crow=0, ldc=31) == -1                          # ldc below the tight one
    assert call(batch=2, st=(0, 0, 0, 0, 32 * 8 - 1)) == -1                         # outputs of the batch overlap
    assert call(off=None) == -1 and call(col=None) == -1 and call(val=None) == -1 and call(B=None) == -1 and call(Cm=None) == -1
    assert call(m=0, bnnz=0) == 0 and call(n=0) == 0                                 # nothing to do: no launch
    assert call(m=1 << 32, k=1 << 32) == -1


def test_workspace_bytes(built_lib):
    """two carry slots of bs x n accumulators per chunk of ch stored blocks, per batch matrix"""
    lib = load(built_lib)
    P = R.params(lib)
    for t, m, n, bs, bnnz, batch in ((F16, 4096, 64, 64, 640, 1), (F64, 4096, 64, 64, 640, 1), (F16, 4096, 64, 64, 640, 16),
                                     (BF16, 16384, 128, 16, 100000, 1), (F32, 64, 8, 4, 3, 2)):
        ch = R.chunk(m // bs, bnnz, P, bs, n, batch)
        want = 2 * (-(-bnnz // ch)) * bs * n * (8 if t == F64 else 4) * batch
        assert lib.b200spmm_bsr_workspace_bytes(t, m, n, bs, bnnz, batch) == want, (t, m, n, bs, bnnz, batch)
    assert lib.b200spmm_bsr_workspace_bytes(F16, 4096, 64, 64, 0, 1) == 0 and lib.b200spmm_bsr_workspace_bytes(F16, 4096, 0, 64, 9, 1) == 0
    assert lib.b200spmm_bsr_workspace_bytes(F16, 4096, 64, 64, 9, 0) == 0


def test_path_selection(built_lib):
    lib = load(built_lib)
    path = lambda t=F16, bs=32, ar=1, V=4096, B=8192, sbk=64, sbj=1, batch=1, sv=0, sb=0: lib.b200spmm_bsr_path(  # noqa: E731
        t, bs, ar, V, B, sbk, sbj, batch, sv, sb)
    assert path() == 1 and path(t=BF16) == 1
    assert path(sbk=1, sbj=64) == 1                                                  # K-contiguous op(B)
    assert path(t=F32) == 0 and path(t=F64) == 0                                     # FFMA / DFMA
    assert path(bs=8) == 0 and path(bs=24) == 0                                      # bs % 16
    assert path(ar=0) == 0                                                           # column-major blocks
    assert path(V=4098) == 0 and path(B=8194) == 0                                   # misaligned views
    assert path(sbk=63) == 0 and path(sbk=64, sbj=64) == 0                           # odd leading dimension, no contiguous dimension
    assert path(batch=2, sb=64 * 65) == 1 and path(batch=2, sb=7) == 0


def test_params(built_lib):
    P = R.params(load(built_lib))
    assert P["k_slab"] == 16 and P["k_slab"] * P["slabs_per_stage"] >= 64 and P["stages"] >= 2
    assert P["max_rows_per_cta"] % 16 == 0 and P["chunk_min"] >= 1 and P["chunk_factor"] >= 1 and P["target_ctas"] >= 132


def test_sass_of_the_bsr_spmm_kernels(built_lib):
    """the tensor path runs HMMA fed by LDSM (.T for an N-contiguous op(B)) from LDGSTS; the CUDA-core path runs FFMA (DFMA for fp64)
    and no tensor instruction; no kernel spills to local memory"""
    sass = subprocess.check_output(["cuobjdump", "-sass", built_lib], text=True)

    def kernel_sass(pattern):
        m = re.search(r"Function : \S*" + pattern + r".*?(?=Function :|\Z)", sass, re.S)
        assert m, pattern
        return m.group(0)
    for t in ("6__half", "13__nv_bfloat16"):
        for bm in (16, 32, 64):
            for bn in (64, 128):
                for bk in (0, 1):
                    body = kernel_sass(rf"spmm_bsr_mma_kernelI{t}Li{bm}ELi{bn}ELb{bk}E")
                    assert "HMMA.16816.F32" in body and "LDGSTS" in body and "LDSM" in body, (t, bm, bn, bk)
                    assert ("LDSM.16.MT88" in body) == (not bk), (t, bm, bn, bk)
                    assert "STL" not in body and "LDL" not in body, (t, bm, bn, bk)
        body = kernel_sass(rf"spmm_bsr_fma_kernelI{t}fEE")
        assert "HMMA" not in body and "FFMA" in body and "STL" not in body
    f32, f64 = kernel_sass(r"spmm_bsr_fma_kernelIffEE"), kernel_sass(r"spmm_bsr_fma_kernelIddEE")
    assert "FFMA" in f32 and "HMMA" not in f32 and "STL" not in f32
    assert "DFMA" in f64 and "DMMA" not in f64 and "STL" not in f64
    assert "HMMA.16816.F32.BF16" in kernel_sass(r"spmm_bsr_mma_kernelI13__nv_bfloat16Li64ELi128ELb0E")
