"""CPU: the half-precision CSR SpMV additions to libb200spmv.so without a device -- symbols, the int64 reference and its precondition,
the fp32 restatement of the summation, both walks' write-once properties, the route table (by shape and over real descriptors), host-side
argument rejection, workspace bytes, params, and what the kernels compile to."""
import ctypes as C
import os
import re
import subprocess
import sys
import textwrap

import numpy as np
import pytest

from cudalibrarysamples_b200.lib import load
from oracle import spmv_csr16_ref as R
from test_abi import declared_symbols, exported

REAL = "/usr/local/cuda/lib64/libcusparse.so.12"
NEW = ["b200spmv_csr16", "b200spmv_csr16_workspace_bytes", "b200spmv_csr16_path", "b200spmv_csr16_params", "b200spmv_csr16_route"]
F32, F64, F16, BF16, C32, I8 = 0, 1, 2, 14, 4, 3
CSR, COO, SELL, CSC, BSR = 1, 2, 9, 3, 5
NT, TR, CT = 0, 1, 2
I32, I64 = 2, 3
DEFAULT, COO_ALG1, CSR_ALG1, CSR_ALG2, COO_ALG2, SELL_ALG1 = 0, 1, 2, 3, 4, 5
FORWARD, HALF16 = 0, 3


def native():
    from scripts.spmv_csr16_bench import NATIVE
    return eval(NATIVE)


def test_header_declares_and_library_exports_the_csr16_spmv_symbols(built_lib):
    names = declared_symbols()
    have = exported(built_lib)
    for n in NEW:
        assert n in names and n in have, n


@pytest.mark.parametrize("base", [0, 1])
def test_int64_reference_matches_scipy_and_checks_its_precondition(base):
    import scipy.sparse as sp
    lengths = [3, 0, 7, 1, 0, 12]
    off, col = R.pattern(lengths, 20, seed=1, base=base)
    val, x, y0 = R.values(6, 20, len(col), seed=2)
    A = sp.csr_matrix((val, col - base, off - base), shape=(6, 20))
    assert np.array_equal(A @ x, R.products(off, col, val, x, base))
    assert np.array_equal(R.reference_int(off, col, val, x, y0, -2.0, 0.5, "f16", base), -2.0 * (A @ x) + 0.5 * y0)
    assert np.array_equal(R.reference_int(off, col, val, x, y0 * np.nan, 1.0, 0.0, "bf16", base), A @ x)
    with pytest.raises(AssertionError):
        R.reference_int(off, col, np.abs(val), np.full_like(x, 300), y0, 1.0, 0.0, "bf16", base)   # 300 * 12 > bf16's 256
    with pytest.raises(AssertionError):
        R.reference_int(off, col, val, x, y0, 3.0, 0.0, "f32", base)                              # alpha not a power of two
    with pytest.raises(AssertionError):
        R.reference_int(off, col, val, np.full_like(x, 1 << 23), y0, 1.0, 0.0, "f32", base)       # sums past 2^24


@pytest.mark.parametrize("kind", ["f16", "bf16"])
def test_fp32_restatement_agrees_with_fp64(kind):
    """random data: the restated fp32 sums are within the fp32 dot-product bound of the fp64 sums of the same 16-bit inputs"""
    import torch
    dt = torch.float16 if kind == "f16" else torch.bfloat16
    lengths = [0, 1, 255, 256, 257, 511, 513, 5, 3000, 0, 17]
    off, col = R.pattern(lengths, 4000, seed=3)
    rng = np.random.default_rng(4)
    val = torch.from_numpy(rng.uniform(-1, 1, len(col))).to(dt).double().numpy()
    x = torch.from_numpy(rng.uniform(-1, 1, 4000)).to(dt).double().numpy()
    acc = R.accumulate_f32(off, col, val, x, 256, 8)
    rows = np.repeat(np.arange(len(lengths)), np.diff(off))
    exact, mag = np.zeros(len(lengths)), np.zeros(len(lengths))
    np.add.at(exact, rows, val * x[col])
    np.add.at(mag, rows, np.abs(val * x[col]))
    assert acc.dtype == np.float32
    assert (np.abs(acc.astype(np.float64) - exact) <= np.diff(off) * 2.0 ** -24 * mag + 1e-300).all()
    assert acc[0] == 0 and acc[9] == 0 and not np.signbit(acc[0])
    # integer data: the restatement is exact
    ival, ix, _ = R.values(len(lengths), 4000, len(col), seed=5)
    assert np.array_equal(R.accumulate_f32(off, col, ival, ix, 256, 8), R.products(off, col, ival, ix))


def test_fp32_restatement_pins_the_order():
    """a run's sum, then the runs of a piece, then the pieces of a row, each from 0, in order: 2^24 + 1 + 1 ... shows the order"""
    E, Rn = 256, 8
    big = 2.0 ** 24
    # one row of 2E + 3 entries: its first product is 2^24, every other 1; in fp32 1 + 2^24 rounds back to 2^24 (ties to even),
    # while 1 + 1 + ... + 1 (a run: 8) then added to 2^24 is exact
    n = 2 * E + 3
    val = np.ones(n)
    val[0] = big
    x = np.ones(1)
    acc = R.accumulate_f32([0, n], np.zeros(n, np.int64), val, x, E, Rn)
    # run 0 = 2^24 + 7 ones, each lost to rounding: 2^24; the other runs are exact; piece 0 = 2^24 + 31 runs of 8 = 2^24 + 248;
    # piece 1 = 256; piece 2 = 3
    assert acc[0] == np.float32(big + 248 + 256 + 3)


def structural(off, E, split):
    writes, reads, pieces = R.walk(off, E, split=split)
    m, nnz = len(off) - 1, int(off[-1])
    ys = sorted(w[1] for w in writes if w[0] == "y")
    assert ys == list(range(m)), (split, ys[:20])                                      # every row written once
    slots = [w[1] for w in writes if w[0] == "carry"]
    assert len(slots) == len(set(slots))                                               # every slot written once
    assert all(s < 2 * max(1, -(-nnz // E)) for s in slots)
    covered = sorted((p[1], p[2]) for p in pieces)
    assert [e for s, t in covered for e in range(s, t)] == list(range(nnz))            # every entry in exactly one piece that counts
    for r, s, e, _ in pieces:
        assert off[r] <= s < e <= off[r + 1] and e - s <= E and (s // E) == ((e - 1) // E)   # a piece lies inside one chunk
    if split:
        assert sorted(x[1] for x in reads) == sorted(slots)                            # every slot read once
        for r in range(m):
            mine = [x for x in reads if x[2] == r]
            if mine:
                rs, re = int(off[r]), int(off[r + 1])
                c = rs // E
                want = [R.slot("out", c)] + [R.slot("in", c2) for c2 in range(c + 1, -(-re // E))]
                assert [x[1] for x in mine] == want and {x[3] for x in mine} == {c}    # one fix-up, at the row's first chunk, in order
                assert [w[2] for w in writes if w[0] == "y" and w[1] == r] == [("fixup", c)]
    # the pieces of each row, in the order it adds them, are its chunk intersections in ascending order
    order = {}
    for r, s, e, _ in pieces:
        order.setdefault(r, []).append((s, e))
    return {r: sorted(v) for r, v in order.items()}, pieces


def patterns(E):
    return {
        "edges": [0, 1, E - 1, E, E + 1, 0, 2 * E - 1, 2 * E + 1, 3, E, 0, 2 * E - 1, 2 * E + 1, 1],
        "long": [5, 40 * E + 17, 0, 2, E + 1],
        "all-empty": [0] * 100,
        "one-row": [3 * E + 7],
        "one-row-short": [3],
        "trailing-empty": [E, E, 0, 0, 0],
        "many-short": [1, 2, 3, 0, 30, 31, 32, 33] * 40,
    }


@pytest.mark.parametrize("name", sorted(patterns(256)))
def test_walk_properties(built_lib, name):
    E = R.params(load(built_lib))["chunk"]
    lengths = patterns(E)[name]
    off = np.concatenate([[0], np.cumsum(lengths)]).astype(np.int64)
    split_order, split_pieces = structural(off, E, True)
    unsplit_order, unsplit_pieces = structural(off, E, False)
    assert split_order == unsplit_order                                 # the same pieces: the same summation order, the same bits
    for r, ps in split_order.items():
        assert [s // E for s, _ in ps] == list(range(ps[0][0] // E, (ps[-1][1] - 1) // E + 1))
    if name == "long":                                                  # the split walk spreads the long row over 41 warps
        assert len({p[3] for p in split_pieces if p[0] == 1}) == 41
        assert len({p[3] for p in unsplit_pieces if p[0] == 1}) == 1


def route(L, fmt=CSR, op=NT, alg=DEFAULT, off=I32, col=I32, a=F16, x=None, y=None, compute=F32, rows=10 << 20, cols=10 << 20,
          nnz=160 << 20):
    x = a if x is None else x
    y = a if y is None else y
    return L.b200spmv_route(fmt, op, alg, off, col, a, x, y, compute, C.c_int64(rows), C.c_int64(cols), C.c_int64(nnz))


def test_route_by_shape(built_lib):
    L = load(built_lib)
    nat = native()
    shapes = [(1 << 20, 16 << 20), (1 << 20, 4 << 20), (1 << 20, 3 << 20), (1 << 16, 1 << 20), (10 << 20, 160 << 20), (10 << 20, (160 << 20) + 5), (10 << 20, 170 << 20),
              (8192 * 8192, 5 * 8192 * 8192 - 4 * 8192), (256 ** 3, 7 * 256 ** 3 - 6 * 256 ** 2), ((1 << 20) - 1, 16 << 20)]
    seen = set()
    for vt, yt in ((F16, F16), (F16, F32), (BF16, BF16), (BF16, F32)):
        for rows, nnz in shapes:
            want = HALF16 if nat(vt, yt, rows, rows, nnz) else FORWARD
            seen.add(want)
            for alg in (DEFAULT, CSR_ALG1, CSR_ALG2):
                assert route(L, a=vt, y=yt, rows=rows, cols=rows, nnz=nnz, alg=alg) == want, (vt, yt, rows, nnz, alg)
    assert HALF16 in seen and FORWARD in seen
    ok = dict(rows=10 << 20, cols=10 << 20, nnz=160 << 20)
    assert nat(F16, F16, **{k: v for k, v in ok.items()})
    # outside the class: forwarded, as before
    assert route(L, compute=F16, y=F16, **ok) == FORWARD                              # fp16 compute
    assert route(L, a=BF16, compute=BF16, **ok) == FORWARD
    assert route(L, a=F16, y=BF16, **ok) == FORWARD and route(L, a=BF16, y=F16, **ok) == FORWARD   # mixed 16-bit pairs
    assert route(L, a=F16, x=BF16, y=F32, **ok) == FORWARD and route(L, a=F16, x=F32, y=F32, **ok) == FORWARD
    assert route(L, op=TR, **ok) == FORWARD and route(L, op=CT, **ok) == FORWARD     # opA T / C
    assert route(L, off=I64, col=I64, **ok) == FORWARD and route(L, col=I64, **ok) == FORWARD   # 64-bit indices
    assert route(L, fmt=COO, **ok) == FORWARD and route(L, fmt=SELL, **ok) == FORWARD            # other formats
    assert route(L, fmt=CSC, **ok) == FORWARD and route(L, fmt=BSR, **ok) == FORWARD
    for alg in (COO_ALG1, COO_ALG2, SELL_ALG1):                                       # other algorithms
        assert route(L, alg=alg, **ok) == FORWARD, alg
    assert route(L, a=I8, x=I8, y=F32, **ok) == FORWARD and route(L, a=C32, compute=C32, **ok) == FORWARD
    assert route(L, compute=F64, **ok) == FORWARD
    assert route(L, rows=1 << 31, cols=1 << 20, nnz=16 << 31) == FORWARD               # past int32
    # the fp32 / fp64 table is untouched
    assert route(L, a=F32, y=F32, compute=F32, **ok) == 1 and route(L, a=F64, y=F64, compute=F64, **ok) == 1


ROUTE = textwrap.dedent("""
    import ctypes as C, os, sys
    sys.path.insert(0, os.path.dirname(os.path.dirname(sys.argv[1])))     # the repository: argv[1] is its built library
    from cudalibrarysamples_b200.lib import load
    real = C.CDLL(sys.argv[2], mode=C.RTLD_GLOBAL)
    shim = load(sys.argv[1])
    I32, I64 = 2, 3
    F32, F64, F16, BF16, I8 = 0, 1, 2, 14, 3
    NT, TR, CT = 0, 1, 2
    buf = (C.c_double * 64)()
    idx = (C.c_int * 64)()

    def csr(rows, cols, nnz, vt=F16, it=I32, lib=shim, coo=False):
        d = C.c_void_p()
        if coo:
            assert lib.cusparseCreateCoo(C.byref(d), C.c_int64(rows), C.c_int64(cols), C.c_int64(nnz), idx, idx, buf, it, 0, vt) == 0
        else:
            assert lib.cusparseCreateCsr(C.byref(d), C.c_int64(rows), C.c_int64(cols), C.c_int64(nnz), idx, idx, buf, it, it, 0, vt) == 0
        return d

    def vec(n, vt, lib=shim):
        d = C.c_void_p()
        assert lib.cusparseCreateDnVec(C.byref(d), C.c_int64(n), buf, vt) == 0
        return d

    forward = sys.argv[3] == "forward"
    for vt, yt in ((F16, F16), (F16, F32), (BF16, BF16), (BF16, F32)):
        for rows, per in ((1 << 16, 16), (1 << 20, 3), (1 << 20, 4), (1 << 20, 16), (10 << 20, 16)):
            nnz = rows * per
            a, x, y = csr(rows, rows, nnz, vt), vec(rows, vt), vec(rows, yt)
            want = 0 if forward else shim.b200spmv_route(1, NT, 0, I32, I32, vt, vt, yt, F32, rows, rows, nnz)
            for alg in (0, 2, 3):
                assert shim.b200spmv_csr16_route(a, x, y, NT, F32, alg) == want, (vt, yt, rows, per, alg)
            assert shim.b200spmv_csr16_route(csr(rows, rows, nnz, vt, lib=real), x, y, NT, F32, 0) == want   # created behind our back
            assert shim.b200spmv_csr16_route(a, x, y, TR, F32, 0) == 0 and shim.b200spmv_csr16_route(a, x, y, CT, F32, 0) == 0
            assert shim.b200spmv_csr16_route(a, x, y, NT, vt, 0) == 0                      # 16-bit compute
            assert shim.b200spmv_csr16_route(a, x, y, NT, F32, 1) == 0                     # COO_ALG1
            assert shim.b200spmv_csr16_route(csr(rows, rows, nnz, vt, it=I64), x, y, NT, F32, 0) == 0
            assert shim.b200spmv_csr16_route(csr(rows, rows, nnz, vt, coo=True), x, y, NT, F32, 0) == 0
            other = BF16 if vt == F16 else F16
            assert shim.b200spmv_csr16_route(a, x, vec(rows, other), NT, F32, 0) == 0      # y of the other 16-bit type
            assert shim.b200spmv_csr16_route(a, vec(rows, other), y, NT, F32, 0) == 0      # x of the other type
            assert shim.b200spmv_csr16_route(None, x, y, NT, F32, 0) == 0
    # fp32 / fp64 descriptors keep their path
    n = 1 << 20
    want = 0 if forward else 1
    assert shim.b200spmv_csr16_route(csr(n, n, 16 * n, F32), vec(n, F32), vec(n, F32), NT, F32, 0) == want
    assert shim.b200spmv_csr16_route(csr(n, n, 16 * n, F64), vec(n, F64), vec(n, F64), NT, F64, 0) == want
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
    one = C.c_float(1.0)
    dummy = (C.c_int * 64)()
    p, o = C.addressof(dummy), C.addressof(one)

    def call(at=F16, yt=F16, m=32, k=32, nnz=2, off=p, col=p, val=p, base=0, alpha=o, beta=o, x=p, y=p):
        return lib.b200spmv_csr16(None, at, yt, m, k, nnz, off, col, val, base, alpha, beta, 0, x, y, None, 0)
    assert call(at=F32, yt=F32) == -1 and call(at=F64, yt=F64) == -1 and call(at=I8) == -1     # fp32 / fp64 are the other kernels'
    assert call(yt=BF16) == -1 and call(at=BF16, yt=F16) == -1 and call(yt=F64) == -1          # mixed 16-bit pairs
    assert call(m=-1) == -1 and call(k=-1) == -1 and call(nnz=-1) == -1
    assert call(nnz=32 * 32 + 1) == -1                                                        # more entries than the matrix holds
    assert call(base=2) == -1 and call(alpha=None) == -1 and call(beta=None) == -1
    assert call(off=None) == -1 and call(col=None) == -1 and call(val=None) == -1 and call(x=None) == -1 and call(y=None) == -1
    assert call(m=1 << 31, k=1) == -1 and call(k=1 << 31) == -1 and call(m=1 << 20, k=1 << 20, nnz=1 << 31) == -1
    assert call(m=0, nnz=0) == 0 and call(m=0, nnz=0, y=None, off=None) == 0                 # nothing to do: no launch


def test_workspace_bytes_params_and_path(built_lib):
    lib = load(built_lib)
    P = R.params(lib)
    E = P["chunk"]
    assert E % 256 == 0 and P["run"] == 8 and P["warps"] >= 1
    ws = lib.b200spmv_csr16_workspace_bytes
    for rows, nnz in ((1 << 20, 16 << 20), (5, 1), (3, E), (3, E + 1), (7, 40 * E + 17)):
        assert ws(rows, nnz) == 2 * (-(-nnz // E)) * 4, (rows, nnz)
    assert ws(0, 0) == 0 and ws(10, 0) == 0
    path = lib.b200spmv_csr16_path
    assert path(4096, 4096) == 2 and path(4096 + 8, 4096 + 4) == 2
    assert path(4096 + 4, 4096) == 1 and path(4096, 4096 + 2) == 1                          # views misaligned by one element


def test_sass_of_the_csr16_spmv_kernels(built_lib):
    """64-bit no-allocate column loads and 32-bit value pairs on the paired path, x through the read-only path, no atomics, no tensor
    instruction, no local memory"""
    sass = subprocess.check_output(["cuobjdump", "-sass", built_lib], text=True)
    bodies = {m.group(1): m.group(2) for m in re.finditer(r"Function : (\S*spmv_csr16_\S*)(.*?)(?=Function :|\Z)", sass, re.S)}
    assert len([k for k in bodies if "chunk_kernel" in k]) == 4 and len([k for k in bodies if "fixup_kernel" in k]) == 2, sorted(bodies)
    for name, body in bodies.items():
        for bad in ("ATOM", "RED.", "HMMA", "STL", "LDL"):
            assert bad not in body, (name, bad)
    for t in ("6__half", "13__nv_bfloat16"):
        paired = bodies[f"_ZN4b20023spmv_csr16_chunk_kernelI{t}Li2EEEvNS_13SpmvCsr16ArgsENS_7ScalarsIfEE"]
        assert re.search(r"LDG\.E\.NA\.64\.CONSTANT", paired), t                            # two columns per lane
        assert re.search(r"LDG\.E\.NA\.CONSTANT ", paired), t                               # two 16-bit values per lane
        assert re.search(r"LDG\.E\.U16\.CONSTANT", paired), t                               # x: read-only, L1-cached
        scalar = bodies[f"_ZN4b20023spmv_csr16_chunk_kernelI{t}Li1EEEvNS_13SpmvCsr16ArgsENS_7ScalarsIfEE"]
        assert re.search(r"LDG\.E\.NA\.U16\.CONSTANT", scalar) and not re.search(r"LDG\.E\.NA\.64", scalar), t
