"""GPU: the half-precision CSR SpMM (spmm_csr16.cu) bit for bit against the int64 reference on integer data, over every type pair,
B / C order, op(B), N edge, index base, scalar placement, padded and misaligned views, and row lengths around the lane, piece and split
edges; both walks, repeats and graph replays bit-identical; NaN guards; parity with the closed library; and the shim's routing."""
import ctypes as C
import textwrap

import numpy as np
import pytest
import torch

from oracle import spmm_csr16_ref as R

pytestmark = pytest.mark.gpu

NT, TR = 0, 1
ROW, COL = 2, 1
VT = {torch.float32: 0, torch.float16: 2, torch.bfloat16: 14}
KIND = {torch.float32: "f32", torch.float16: "f16", torch.bfloat16: "bf16"}
TYPES = [(torch.float16, torch.float16), (torch.float16, torch.float32), (torch.bfloat16, torch.bfloat16), (torch.bfloat16, torch.float32)]
LAYOUTS = {"rowrow": dict(opB=NT, ob=ROW, oc=ROW), "colcol": dict(opB=NT, ob=COL, oc=COL), "rowcol": dict(opB=NT, ob=ROW, oc=COL),
           "colrow": dict(opB=NT, ob=COL, oc=ROW), "T-rowrow": dict(opB=TR, ob=ROW, oc=ROW), "T-colcol": dict(opB=TR, ob=COL, oc=COL)}
DEV = "cuda"


@pytest.fixture(scope="module")
def L():
    from cudalibrarysamples_b200 import lib
    return lib.shim()


def stored_b(b, opB, order, pad, dt, shift, nan_rows=None):
    """device buffer holding the matrix whose op() is b (k x n), NaN in the ld padding (and in op(B) rows nan_rows), starting `shift`
    elements into the allocation; returns (buffer, view pointer, sbk, sbj) with op(B)(k, j) = view[k * sbk + j * sbj]"""
    bb = b.astype(np.float64).copy()
    if nan_rows is not None:
        bb[nan_rows] = np.nan
    X = bb if opB == NT else bb.T
    r, c = X.shape
    ld = (c if order == ROW else r) + pad
    buf = torch.full((shift + (r if order == ROW else c) * ld + 8,), float("nan"), dtype=torch.float64)
    body = buf[shift:shift + (r if order == ROW else c) * ld]
    if order == ROW:
        body.view(r, ld)[:, :c] = torch.from_numpy(X)
        sr, sc = ld, 1
    else:
        body.view(c, ld)[:, :r] = torch.from_numpy(X.T.copy())
        sr, sc = 1, ld
    s1, s2 = (sr, sc) if opB == NT else (sc, sr)
    d = buf.to(dt).to(DEV)
    return d, d.data_ptr() + 2 * shift, s1, s2


def run(L, dt, ct, m, off, col, val, b, c0, alpha=1.0, beta=0.0, opB=NT, ob=ROW, oc=ROW, base=0, pad=0, shift=0, on_device=False,
        split=True, nan_rows=None):
    """one b200spmm_csr16 call; returns C as float64 m x n numpy.  C0 is NaN where beta == 0."""
    k, n = b.shape
    Bb, pB, sbk, sbj = stored_b(b, opB, ob, pad, dt, shift, nan_rows)
    ldc = (n if oc == ROW else m) + pad
    Cb = torch.full(((m if oc == ROW else n) * ldc + shift,), float("nan"), dtype=torch.float64)
    if beta != 0:
        body = Cb[shift:]
        view = body.view(m, ldc)[:, :n] if oc == ROW else body.view(n, ldc)[:, :m].T
        view.copy_(torch.from_numpy(c0.astype(np.float64)))
    Cd = Cb.to(ct).to(DEV)
    V = torch.tensor(np.asarray(val, np.float64), dtype=dt, device=DEV)
    offd = torch.tensor(off, dtype=torch.int32, device=DEV)
    cold = torch.tensor(col, dtype=torch.int32, device=DEV)
    if on_device:
        al, be = torch.tensor([alpha], dtype=torch.float32, device=DEV), torch.tensor([beta], dtype=torch.float32, device=DEV)
        pa, pb = al.data_ptr(), be.data_ptr()
    else:
        al, be = C.c_float(alpha), C.c_float(beta)
        pa, pb = C.addressof(al), C.addressof(be)
    wsb = L.b200spmm_csr16_workspace_bytes(k, n, len(col), sbk, sbj)
    ws = torch.full((max(wsb, 16),), 0x7F, dtype=torch.uint8, device=DEV)
    rc = L.b200spmm_csr16(torch.cuda.current_stream().cuda_stream, VT[dt], VT[ct], m, k, n, len(col), offd.data_ptr(), cold.data_ptr(),
                          V.data_ptr(), base, pa, pb, int(on_device), pB, sbk, sbj, Cd.data_ptr() + Cd.element_size() * shift, ldc,
                          int(oc == ROW), ws.data_ptr() if split else None, wsb if split else 0)
    torch.cuda.synchronize()
    assert rc == 0
    out = Cd.double().cpu()[shift:]
    out = out.view(m, ldc)[:, :n] if oc == ROW else out.view(n, ldc)[:, :m].T
    return out.numpy().copy()


def check(L, dt, ct, off, col, val, b, c0, alpha=1.0, beta=0.0, base=0, **kw):
    m = len(off) - 1
    ref = R.reference_int(off, col, val, b, c0, alpha, beta, KIND[ct], base)
    got = {}
    for split in (True, False):
        got[split] = run(L, dt, ct, m, off, col, val, b, c0, alpha, beta, base=base, split=split, **kw)
        assert np.array_equal(got[split], ref), (dt, ct, split, kw, np.nanmax(np.abs(got[split] - ref)))


def case(lengths, k, n, seed=1, base=0):
    off, col = R.pattern(lengths, k, seed, base)
    val, b, c0 = R.values(len(lengths), k, n, len(col), seed + 1)
    return off, col, val, b, c0


@pytest.mark.parametrize("dt,ct", TYPES, ids=lambda t: str(t)[6:])
@pytest.mark.parametrize("layout", sorted(LAYOUTS))
def test_types_layouts_and_n_edges(L, dt, ct, layout):
    for n in (1, 7, 8, 31, 32, 33, 64, 65, 128, 129, 256):
        off, col, val, b, c0 = case([3, 0, 1, 9, 33, 2, 0, 40, 5] * 4, 80, n, seed=n)
        check(L, dt, ct, off, col, val, b, c0, 2.0 if ct != torch.bfloat16 else 1.0, 0.5, **LAYOUTS[layout])


@pytest.mark.parametrize("dt,ct", TYPES, ids=lambda t: str(t)[6:])
def test_base_one_device_scalars_padding_and_misaligned_views(L, dt, ct):
    off, col, val, b, c0 = case([3, 0, 1, 9, 33, 2, 0, 40, 5] * 4, 80, 72, base=1)
    for layout in ("rowrow", "colcol", "T-rowrow"):
        kw = LAYOUTS[layout]
        check(L, dt, ct, off, col, val, b, c0, -2.0, 0.5, base=1, **kw)
        check(L, dt, ct, off, col, val, b, c0, -2.0, 0.5, base=1, on_device=True, **kw)
        check(L, dt, ct, off, col, val, b, c0, 2.0, 0.0, base=1, on_device=True, **kw)       # beta = 0 on a NaN C
        check(L, dt, ct, off, col, val, b, c0, 1.0, 1.0, base=1, pad=8, **kw)
        check(L, dt, ct, off, col, val, b, c0, 1.0, 1.0, base=1, pad=3, **kw)               # an odd leading dimension
        check(L, dt, ct, off, col, val, b, c0, 1.0, 1.0, base=1, shift=1, **kw)             # views misaligned by one element


def test_path_of_the_views(L):
    for n, pad, shift, want in ((128, 0, 0, 4), (256, 8, 0, 8), (64, 0, 0, 2), (128, 3, 0, 1), (128, 0, 1, 1), (32, 0, 0, 1)):
        b = np.zeros((16, n), np.int64)
        _, p, sbk, sbj = stored_b(b, NT, ROW, pad, torch.float16, shift)
        assert L.b200spmm_csr16_path(n, p, sbk, sbj) == want, (n, pad, shift)


@pytest.mark.parametrize("dt,ct", [(torch.float16, torch.float32), (torch.bfloat16, torch.bfloat16)], ids=["f16-f32", "bf16"])
@pytest.mark.parametrize("layout", ["rowrow", "colcol"])
def test_row_lengths_around_the_lane_piece_and_split_edges(L, dt, ct, layout):
    P = R.params(L)
    p, le = P["piece"], P["lane_entries"]
    lengths = [0, 1, le - 1, le, le + 1, 2 * le + 1, p - 1, p, p + 1, 0, 2 * p - 1, 2 * p, 2 * p + 1, 3 * p + le + 1, 5, 0]
    k = 4 * p
    off, col = R.pattern(lengths, k, 3)
    rng = np.random.default_rng(4)
    val = rng.choice([-1, 1], len(col))
    b = rng.integers(-1, 2, (k, 40))
    if ct == torch.bfloat16:                                   # bf16 holds integers to 256: a sparser B
        b = np.where(rng.random((k, 40)) < 0.05, b, 0)
    check(L, dt, ct, off, col, val, b, None, **LAYOUTS[layout])   # fp16 -> fp32: sums up to 3 * p + 33 in magnitude


def test_one_row_of_forty_thousand_entries(L):
    """a single row split into ~80 pieces spread over as many warps: exact, and both walks identical"""
    n, k = 64, 50000
    off, col = R.pattern([3, 40000, 0, 7], k, 5)
    rng = np.random.default_rng(6)
    val = rng.choice([-1, 1], len(col))
    b = np.where(rng.random((k, n)) < 0.04, rng.choice([-1, 1], (k, n)), 0)
    check(L, torch.float16, torch.float16, off, col, val, b, None)
    check(L, torch.bfloat16, torch.float32, off, col, val, b, None, **LAYOUTS["colcol"])


@pytest.mark.parametrize("dt", [torch.float16, torch.bfloat16])
def test_nan_guards(L, dt):
    """NaN in rows of op(B) no entry references, in ld padding, and in C with beta = 0 never reaches C; NaN in row 0 of op(B) reaches
    exactly the rows that store column 0"""
    k, n = 60, 40
    lengths = [4, 0, 3, 6, 1, 2]
    off, col = R.pattern(lengths, 30, 7)                                  # columns below 30 only
    val, b, c0 = R.values(len(lengths), k, n, len(col), 8)
    val = np.where(val == 0, 1, val)
    unused = sorted(set(range(k)) - set(col.tolist()))
    ref = R.reference_int(off, col, val, b, c0, 1.0, 0.0, KIND[dt])
    for name, kw in LAYOUTS.items():
        for split in (True, False):
            got = run(L, dt, dt, len(lengths), off, col, val, b, c0, 1.0, 0.0, pad=8, nan_rows=unused, split=split, **kw)
            assert np.array_equal(got, ref), (name, split)
    col0 = col + 1                                                         # columns 1 .. 30, and 0 in rows 0 and 3 only
    col0[off[0]] = col0[off[3]] = 0
    stores0 = np.isin(np.arange(len(lengths)), [0, 3])
    for split in (True, False):
        got = run(L, dt, dt, len(lengths), off, col0, val, b, c0, 1.0, 0.0, nan_rows=[0], split=split)
        assert (np.isnan(got).any(axis=1) == stores0).all() and np.isnan(got[stores0]).all(), split


def random_call(L, dt, ct, lengths, n, k, order, seed=3):
    g = torch.Generator(device=DEV).manual_seed(seed)
    off, col = R.pattern(lengths, k, seed)
    m = len(lengths)
    V = torch.randn(len(col), device=DEV, generator=g).to(dt)
    B = torch.randn(k, n, device=DEV, generator=g).to(dt)
    if order == COL:
        B = B.t().contiguous()
    sbk, sbj = (n, 1) if order == ROW else (1, k)
    offd, cold = torch.tensor(off, dtype=torch.int32, device=DEV), torch.tensor(col, dtype=torch.int32, device=DEV)
    Cm = torch.zeros(m * n, dtype=ct, device=DEV)
    wsb = L.b200spmm_csr16_workspace_bytes(k, n, len(col), sbk, sbj)
    ws = torch.empty(max(wsb, 16), dtype=torch.uint8, device=DEV)
    one, zero = C.c_float(1.0), C.c_float(0.0)

    def call(stream, split=True):
        assert L.b200spmm_csr16(stream.cuda_stream, VT[dt], VT[ct], m, k, n, len(col), offd.data_ptr(), cold.data_ptr(), V.data_ptr(), 0,
                                C.addressof(one), C.addressof(zero), 0, B.data_ptr(), sbk, sbj, Cm.data_ptr(), n if order == ROW else m,
                                int(order == ROW), ws.data_ptr() if split else None, wsb if split else 0) == 0
    return call, Cm


@pytest.mark.parametrize("dt,ct", [(torch.float16, torch.float32), (torch.bfloat16, torch.bfloat16)], ids=["f16-f32", "bf16"])
@pytest.mark.parametrize("order", [ROW, COL])
def test_repeat_graph_replay_and_null_buffer_are_bit_identical(L, dt, ct, order):
    call, Cm = random_call(L, dt, ct, [3, 5000, 0, 700, 1, 1300] * 3, 128, 6000, order)
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        call(s)
    torch.cuda.synchronize()
    first = Cm.clone()
    assert torch.isfinite(first).all()
    for split in (True, True, False, False):
        Cm.fill_(float("nan"))
        with torch.cuda.stream(s):
            call(s, split)
        torch.cuda.synchronize()
        assert torch.equal(Cm, first), split
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph, stream=s):
        call(s)
    for _ in range(3):
        Cm.fill_(float("nan"))
        graph.replay()
        torch.cuda.synchronize()
        assert torch.equal(Cm, first)


@pytest.mark.parametrize("dt,ct", TYPES, ids=lambda t: str(t)[6:])
@pytest.mark.parametrize("order", [ROW, COL])
def test_parity_with_the_closed_library_at_an_rmat_size(L, dt, ct, order):
    """ours and the closed cusparseSpMM on the same buffers, R-MAT 64K x 64K with 16 per row: both within one rounding to C's type
    plus the fp32 dot-product bound of fp64"""
    import scripts.spmm_csr16_bench as SB
    from cudalibrarysamples_b200 import workloads as W
    m = 1 << 16
    off, col, val = W.rmat_csr(m, avg_nnz=16, seed=3, val_seed=4, dtype=torch.float32)
    row = SB.run_case(L, "rmat64k", m, off.int(), col.int(), val.float(), 96, dt, ct, order)
    u = {torch.float16: 2.0 ** -11, torch.bfloat16: 2.0 ** -8, torch.float32: 2.0 ** -24}
    kmax = int((off[1:] - off[:-1]).max())
    tol = kmax * 2.0 ** -24 + u[ct]
    assert row["err_ours"] <= tol, row
    assert row.get("err_closed", 0.0) <= 4 * tol, row


# ------------------------------------------------------------------------------------------------ through the shim
def shim_call(impl, dt, ct, off, col, val, b, c0, order, opB=NT, alg=0, log=False):
    from cudalibrarysamples_b200 import cusparse_api as cs
    api = cs.Api(impl)
    m, (k, n) = len(off) - 1, b.shape
    arr = dict(off=torch.tensor(off, dtype=torch.int32, device=DEV), col=torch.tensor(col, dtype=torch.int32, device=DEV),
               val=torch.tensor(np.asarray(val, np.float64), dtype=dt, device=DEV))
    X = b if opB == NT else b.T
    Bt = torch.tensor(X if order == ROW else X.T.copy(), dtype=dt, device=DEV).contiguous().view(-1)
    Ct = torch.tensor(c0 if order == ROW else c0.T.copy(), dtype=ct, device=DEV).contiguous().view(-1)
    out = cs.spmm(api, m, k, arr, Bt, Ct, 1.0, 1.0, order_b=order, order_c=order, n=n, alg=alg, op_b=opB)
    out = out.double().cpu().numpy()
    return out.reshape(m, n) if order == ROW else out.reshape(n, m).T


SHIM = textwrap.dedent("""
    import ctypes as C, sys
    import torch
    from cudalibrarysamples_b200 import cusparse_api as cs, lib
    L = lib.shim()


    def run(dt, ct, n, m, per, order):
        dt, ct = eval(dt), eval(ct)
        n, m, per, order = int(n), int(m), int(per), int(order)
        g = torch.Generator(device="cuda").manual_seed(n)
        lengths = torch.full((m,), per, dtype=torch.int32, device="cuda")
        lengths[7], lengths[8] = 3000, 0                                     # one row long enough to be split, one empty row
        off = torch.zeros(m + 1, dtype=torch.int32, device="cuda")
        off[1:] = torch.cumsum(lengths, 0)
        nnz = int(off[-1])
        col = torch.randint(0, m, (nnz,), device="cuda", generator=g, dtype=torch.int32)
        rows = torch.repeat_interleave(torch.arange(m, device="cuda"), lengths.long())
        col = col[torch.argsort(rows.long() * m + col.long())].contiguous()
        val = (torch.rand(nnz, device="cuda", generator=g) * 2 - 1).to(dt)
        B = (torch.rand(m * n, device="cuda", generator=g) * 2 - 1).to(dt)
        C0 = (torch.rand(m * n, device="cuda", generator=g) * 2 - 1).to(ct)
        api = cs.Api("b200")
        api.reset_stats()
        got = cs.spmm(api, m, m, dict(off=off, col=col, val=val), B, C0, 1.0, 1.0, order_b=order, order_c=order, n=n)
        st = api.stats()
        sbk, sbj = (n, 1) if order == cs.CUSPARSE_ORDER_ROW else (1, m)
        wsb = L.b200spmm_csr16_workspace_bytes(m, n, nnz, sbk, sbj)
        ws = torch.empty(wsb, dtype=torch.uint8, device="cuda")
        direct = C0.clone()
        one = C.c_float(1.0)
        assert L.b200spmm_csr16(torch.cuda.current_stream().cuda_stream, cs._VT[dt], cs._VT[ct], m, m, n, nnz, off.data_ptr(), col.data_ptr(),
                                val.data_ptr(), 0, C.addressof(one), C.addressof(one), 0, B.data_ptr(), sbk, sbj, direct.data_ptr(),
                                n if order == cs.CUSPARSE_ORDER_ROW else m, int(order == cs.CUSPARSE_ORDER_ROW), ws.data_ptr(), wsb) == 0
        torch.cuda.synchronize()
        closed = cs.spmm(cs.Api("cusparse"), m, m, dict(off=off, col=col, val=val), B, C0, 1.0, 1.0, order_b=order, order_c=order, n=n)
        row = order == cs.CUSPARSE_ORDER_ROW
        mat = lambda x: x.view(m, n) if row else x.view(n, m).t()                     # noqa: E731
        A = torch.sparse_csr_tensor(off, col, val.float().abs(), (m, m))
        bound = (A @ mat(B.float().abs())).double() + mat(C0.double().abs())           # |A| . |op(B)| + |beta C0|
        diff = mat((closed.double() - got.double()).abs())
        err = (diff / (bound + 1e-30)).max().item()
        print("native", st["native"], "forwarded", st["forwarded"], "equal", bool(torch.equal(got, direct)), "closed_err", err, flush=True)
        print(f"[class done {n} {order}]", file=sys.stderr, flush=True)


    for cls in sys.argv[1:]:
        run(*cls.split(","))
""")


def native_classes():
    """the routed classes (type pair, N, order) with the smallest matrix of each, from the route's table"""
    from scripts.spmm_csr16_bench import NATIVE
    native = eval(NATIVE)
    out = {}
    for dt, ct in TYPES:
        for n in (32, 64, 128, 256):
            for order in (ROW, COL):
                for m, per in ((1 << 20, 16), (2 << 20, 32)):
                    if native(VT[dt], VT[ct], n, m, m * per, order) and (dt, ct, n, order) not in out:
                        out[(dt, ct, n, order)] = (m, per)
    return out


def test_shim_runs_every_routed_class_natively(L):
    """one cusparseSpMM per routed class (type pair, N and order; the smallest matrix of the class, with a split row and an empty row):
    native with nothing forwarded, the log line names the kernel, bit-identical to b200spmm_csr16 with the same workspace, and within
    the fp32 accumulation bound of the closed library, relative to |A| . |op(B)| + |C0| (on the long row the closed library is off by
    more than one rounding of a 16-bit C)"""
    import os
    import subprocess
    import sys
    classes = native_classes()
    if not classes:
        pytest.skip("no class is routed natively")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    env = dict(os.environ, B200SPMV_LOG="1", PYTHONPATH=root)
    u = {torch.float16: 2.0 ** -11, torch.bfloat16: 2.0 ** -8, torch.float32: 2.0 ** -24}
    args = [f"{dt},{ct},{n},{m},{per},{order}" for (dt, ct, n, order), (m, per) in classes.items()]
    p = subprocess.run([sys.executable, "-c", SHIM, *args], capture_output=True, text=True, timeout=1800, env=env, cwd=root)
    assert p.returncode == 0, p.stdout + p.stderr[-3000:]
    lines = p.stdout.splitlines()
    assert len(lines) == len(args), p.stdout
    for a, line in zip(args, lines):
        out = line.split()
        assert out[:6] == ["native", "1", "forwarded", "0", "equal", "True"], (a, line)
        assert float(out[7]) < 4 * (u[eval(a.split(",")[1])] + 3000 * 2.0 ** -24), (a, line)
    log = p.stderr.split("[class done")
    assert all("[b200spmv] SpMM CSR 16-bit spmm_csr16_kernel split" in chunk for chunk in log[:-1]), p.stderr[-2000:]


def test_forwarded_kinds_are_counted(L):
    """a 16-bit CSR call outside the routed classes (small, mixed orders, opA = T) goes to the closed library, counted, same result"""
    from cudalibrarysamples_b200 import cusparse_api as cs
    off, col, val, b, c0 = case([3, 0, 5, 2], 6, 8)
    b200 = cs.Api("b200")
    for kw in (dict(order=ROW), dict(order=COL), dict(order=ROW, opB=TR)):
        b200.reset_stats()
        got = shim_call("b200", torch.float16, torch.float32, off, col, val, b, c0, **kw)
        st = b200.stats()
        assert st["native"] == 0 and st["forwarded"] == 1, (kw, st)
        assert np.array_equal(got, shim_call("cusparse", torch.float16, torch.float32, off, col, val, b, c0, **kw))
