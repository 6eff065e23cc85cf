"""GPU: the BSR SpMM (spmm_bsr.cu) bit for bit against the int64 reference on integer data, on both paths and both walks, at every
block size, type pair, block order, B / C order, op(B), N edge and block-row edge; batches, scalars, NaN guards, determinism, parity
with the closed library, the shim, and a block-sparse attention head end to end."""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import spmm_bsr_ref as R

pytestmark = pytest.mark.gpu

NT, TR = 0, 1
ROW, COL = 2, 1
VT = {torch.float32: 0, torch.float64: 1, torch.float16: 2, torch.bfloat16: 14}
KIND = {torch.float32: "f32", torch.float64: "f64", torch.float16: "f16", torch.bfloat16: "bf16"}
TYPES = [(torch.float16, torch.float16), (torch.float16, torch.float32), (torch.bfloat16, torch.bfloat16), (torch.bfloat16, torch.float32),
         (torch.float32, torch.float32), (torch.float64, torch.float64)]
DEV = "cuda"


@pytest.fixture(scope="module")
def L():
    from cudalibrarysamples_b200 import lib
    return lib.shim()


def stored_b(b, opB, order, pad, dt, nan_rows=None):
    """device buffer holding the matrix whose op() is b (k x n), NaN in the ld padding (and in op(B) rows nan_rows); returns (buffer,
    sbk, sbj) with op(B)(k, j) = buf[k * sbk + j * sbj]"""
    bb = b.astype(np.float64).copy()
    if nan_rows is not None:
        bb[nan_rows] = np.nan
    X = bb if opB == NT else bb.T
    r, c = X.shape
    ld = (c if order == ROW else r) + pad
    buf = torch.full(((r if order == ROW else c) * ld + 8,), float("nan"), dtype=torch.float64)
    if order == ROW:
        buf[:r * ld].view(r, ld)[:, :c] = torch.from_numpy(X)
        sr, sc = ld, 1
    else:
        buf[:c * ld].view(c, ld)[:, :r] = torch.from_numpy(X.T.copy())
        sr, sc = 1, ld
    s1, s2 = (sr, sc) if opB == NT else (sc, sr)
    return buf.to(dt).to(DEV), s1, s2


def run(L, dt, ct, m, k, bs, off, col, val, b, c0, alpha=1.0, beta=0.0, opB=NT, ob=ROW, oc=ROW, oa="row", base=0, pad=0, on_device=False,
        split=True, nan_c=None, nan_rows=None, ws_bytes=None):
    """one b200spmm_bsr call on integer data; returns (C as float64 m x n numpy, path)"""
    n = b.shape[1]
    Bb, sbk, sbj = stored_b(b, opB, ob, pad, dt, nan_rows)
    ldc = (n if oc == ROW else m) + pad
    Cb = torch.full(((m if oc == ROW else n) * ldc,), float("nan"), dtype=torch.float64)
    if not (nan_c if nan_c is not None else beta == 0):
        view = Cb.view(m, ldc)[:, :n] if oc == ROW else Cb.view(n, ldc)[:, :m].T
        view.copy_(torch.from_numpy(c0.astype(np.float64)))
    Cd = Cb.to(ct).to(DEV)
    V = torch.tensor(val, dtype=dt, device=DEV)
    offd = torch.tensor(off, dtype=torch.int32, device=DEV)
    cold = torch.tensor(col, dtype=torch.int32, device=DEV)
    sdt = torch.float64 if dt == torch.float64 else torch.float32
    if on_device:
        al, be = torch.tensor([alpha], dtype=sdt, device=DEV), torch.tensor([beta], dtype=sdt, device=DEV)
        pa, pb = al.data_ptr(), be.data_ptr()
    else:
        ctyp = C.c_double if dt == torch.float64 else C.c_float
        al, be = ctyp(alpha), ctyp(beta)
        pa, pb = C.addressof(al), C.addressof(be)
    wsb = L.b200spmm_bsr_workspace_bytes(VT[dt], m, n, bs, len(col), 1) if ws_bytes is None else ws_bytes
    ws = torch.full((max(wsb, 16),), 0x7F, dtype=torch.uint8, device=DEV)
    path = L.b200spmm_bsr_path(VT[dt], bs, int(oa == "row"), V.data_ptr(), Bb.data_ptr(), sbk, sbj, 1, 0, 0)
    rc = L.b200spmm_bsr(torch.cuda.current_stream().cuda_stream, VT[dt], VT[ct], m, k, n, bs, len(col), offd.data_ptr(), cold.data_ptr(),
                        V.data_ptr(), base, int(oa == "row"), pa, pb, int(on_device), Bb.data_ptr(), sbk, sbj, Cd.data_ptr(), ldc,
                        int(oc == ROW), 1, 0, 0, 0, 0, 0, ws.data_ptr() if split else None, wsb if split else 0)
    torch.cuda.synchronize()
    assert rc == 0
    out = Cd.double().cpu()
    out = out.view(m, ldc)[:, :n] if oc == ROW else out.view(n, ldc)[:, :m].T
    return out.numpy().copy(), path


def case(bs, nbr, nbc, n, counts=(2, 0, 1, 4), seed=1, base=0):
    off, col = R.pattern(nbr, nbc, list(counts), seed, base)
    val, b, c0 = R.values(nbr * bs, nbc * bs, n, len(col), bs, seed + 1)
    return off, col, val, b, c0


def check(L, dt, ct, bs, off, col, val, b, c0, alpha=1.0, beta=0.0, base=0, oa="row", **kw):
    m, k = (len(off) - 1) * bs, b.shape[0]
    R.check_exact(m, k, bs, off, col, val, b, c0, alpha, beta, KIND[ct], base, oa)
    ref = R.reference(m, k, bs, off, col, val, b, c0, alpha, beta, base, oa)
    paths = set()
    for split in (True, False):
        got, path = run(L, dt, ct, m, k, bs, off, col, val, b, c0, alpha, beta, base=base, oa=oa, split=split, **kw)
        assert np.array_equal(got, ref), (dt, ct, bs, split, kw, np.nanmax(np.abs(got - ref)))
        paths.add(path)
    return paths.pop()


LAYOUTS = {"attention": dict(opB=NT, ob=ROW, oc=ROW), "colmajor": dict(opB=NT, ob=COL, oc=COL), "opBT": dict(opB=TR, ob=ROW, oc=ROW),
           "mixed": dict(opB=TR, ob=COL, oc=COL)}


@pytest.mark.parametrize("dt,ct", TYPES, ids=lambda t: str(t)[6:])
@pytest.mark.parametrize("bs", [2, 4, 8, 16, 32, 64, 128])
@pytest.mark.parametrize("oa", ["row", "col"])
@pytest.mark.parametrize("layout", sorted(LAYOUTS))
def test_types_block_sizes_orders_and_layouts(L, dt, ct, bs, oa, layout):
    nbr, nbc = (5, 4) if bs <= 32 else (3, 3)
    off, col, val, b, c0 = case(bs, nbr, nbc, 40)
    path = check(L, dt, ct, bs, off, col, val, b, c0, 2.0 if ct != torch.bfloat16 else 1.0, 0.5, oa=oa, pad=8, **LAYOUTS[layout])
    assert path == int(dt in (torch.float16, torch.bfloat16) and bs % 16 == 0 and oa == "row")


@pytest.mark.parametrize("dt", [torch.float16, torch.bfloat16, torch.float32, torch.float64])
@pytest.mark.parametrize("layout", ["attention", "colmajor"])
def test_n_edges(L, dt, layout):
    for n in (1, 7, 8, 63, 64, 65, 129):
        off, col, val, b, c0 = case(16, 4, 3, n, counts=(2, 1, 3, 0))
        pad = 8 if dt in (torch.float16, torch.bfloat16) else 3
        check(L, dt, dt, 16, off, col, val, b, c0, 1.0, 1.0, pad=pad, **LAYOUTS[layout])


@pytest.mark.parametrize("dt,bs", [(torch.float16, 16), (torch.bfloat16, 32), (torch.float16, 64), (torch.float32, 4), (torch.float64, 8)])
def test_empty_block_rows_and_a_global_row_long_enough_to_be_split(L, dt, bs):
    nb = 40 if bs <= 16 else 12
    counts = [0, 2, nb, 0, 1, 3, 0, 2, 1, 0]
    off, col, val, b, c0 = case(bs, len(counts), nb, 72, counts=counts)
    assert off[1] == off[0] and off[-1] == off[-2]
    P = R.params(L)
    assert off[3] - off[2] > R.chunk(len(counts), len(col), P, bs, 72)          # the global block-row is cut into pieces
    check(L, dt, dt, bs, off, col, val, b, c0, 1.0, 1.0)
    check(L, dt, dt, bs, off, col, val, b, c0, 2.0, 0.0, nan_c=True)


@pytest.mark.parametrize("dt", [torch.float16, torch.float32])
def test_base_one_and_device_scalars(L, dt):
    off, col, val, b, c0 = case(16, 4, 3, 24, base=1)
    check(L, dt, dt, 16, off, col, val, b, c0, -2.0, 0.5, base=1)
    check(L, dt, dt, 16, off, col, val, b, c0, -2.0, 0.5, base=1, on_device=True)
    check(L, dt, dt, 16, off, col, val, b, c0, 2.0, 0.0, base=1, on_device=True, nan_c=True)


@pytest.mark.parametrize("dt,bs", [(torch.float16, 32), (torch.bfloat16, 16), (torch.float32, 8), (torch.float64, 2)])
def test_nan_guards(L, dt, bs):
    """beta = 0 on a NaN C; NaN in ld padding and in rows of op(B) no stored block references"""
    nb = 5
    off, col = R.pattern(nb, nb, [1, 0, 2, 0], seed=3)
    val, b, c0 = R.values(nb * bs, nb * bs, 24, len(col), bs, seed=4)
    unused = [r for r in range(nb * bs) if r // bs not in set(col.tolist())]
    assert unused
    m = nb * bs
    R.check_exact(m, m, bs, off, col, val, b, c0, 1.0, 0.0, KIND[dt])
    ref = R.reference(m, m, bs, off, col, val, b, c0, 1.0, 0.0)
    for layout in LAYOUTS.values():
        for split in (True, False):
            got, _ = run(L, dt, dt, m, m, bs, off, col, val, b, c0, 1.0, 0.0, pad=8, nan_c=True, nan_rows=unused, split=split, **layout)
            assert np.array_equal(got, ref), (layout, split)


@pytest.mark.parametrize("dt", [torch.float16, torch.bfloat16])
def test_misaligned_views_take_the_cuda_core_path_exactly(L, dt):
    off, col, val, b, c0 = case(32, 3, 3, 40)
    assert check(L, dt, dt, 32, off, col, val, b, c0, 1.0, 1.0, pad=3) == 0        # odd leading dimension
    assert check(L, dt, dt, 32, off, col, val, b, c0, 1.0, 1.0, pad=8) == 1


def run_batch(L, dt, bs, nb, n, batch, share, seed=5, split=True):
    """a strided batch; share: subset of "ocvB" (offsets / columns / values / B shared by the batch).  Returns (got, expected)"""
    m = nb * bs
    offs, cols, vals, Bs, Cs = [], [], [], [], []
    for i in range(batch):
        si = 0 if ("o" in share and "c" in share) else i
        off, col = R.pattern(nb, nb, [2, 1, 0, 3], seed + si)
        if "o" in share and "c" not in share:         # shared offsets, per-matrix columns: same counts, different columns
            assert np.array_equal(off, R.pattern(nb, nb, [2, 1, 0, 3], seed)[0])
        val, _, c0 = R.values(m, m, n, len(col), bs, seed + 10 + (0 if "v" in share else i))
        _, b, _ = R.values(m, m, n, len(col), bs, seed + 20 + (0 if "B" in share else i))
        offs.append(off); cols.append(col); vals.append(val); Bs.append(b); Cs.append(c0)
    bnnz = len(cols[0])
    exp = np.stack([R.reference(m, m, bs, offs[i], cols[i], vals[i], Bs[i], Cs[i], 1.0, 1.0) for i in range(batch)])
    t = lambda x: torch.tensor(np.array(x), device=DEV)  # noqa: E731
    off_d = t(offs[0] if "o" in share else np.concatenate(offs)).int()
    col_d = t(cols[0] if "c" in share else np.concatenate(cols)).int()
    V_d = t(vals[0] if "v" in share else np.concatenate(vals)).to(dt).contiguous()
    B_d = t(Bs[0] if "B" in share else np.stack(Bs)).to(dt).contiguous()
    C_d = t(np.stack(Cs)).to(dt).contiguous()
    one = C.c_double(1.0) if dt == torch.float64 else C.c_float(1.0)
    wsb = L.b200spmm_bsr_workspace_bytes(VT[dt], m, n, bs, bnnz, batch)
    ws = torch.empty(max(wsb, 16), dtype=torch.uint8, device=DEV)
    rc = L.b200spmm_bsr(torch.cuda.current_stream().cuda_stream, VT[dt], VT[dt], m, m, n, bs, bnnz, off_d.data_ptr(), col_d.data_ptr(),
                        V_d.data_ptr(), 0, 1, C.addressof(one), C.addressof(one), 0, B_d.data_ptr(), n, 1, C_d.data_ptr(), n, 1, batch,
                        0 if "o" in share else nb + 1, 0 if "c" in share else bnnz, 0 if "v" in share else bnnz * bs * bs,
                        0 if "B" in share else m * n, m * n, ws.data_ptr() if split else None, wsb if split else 0)
    torch.cuda.synchronize()
    assert rc == 0
    return C_d.double().cpu().numpy(), exp


@pytest.mark.parametrize("dt,bs", [(torch.float16, 16), (torch.bfloat16, 64), (torch.float32, 4)])
@pytest.mark.parametrize("share", ["", "o", "oc", "v", "B", "ocvB"])
def test_strided_batches(L, dt, bs, share):
    for split in (True, False):
        got, exp = run_batch(L, dt, bs, 5, 40, 3, share, split=split)
        assert np.array_equal(got, exp), (share, split)


def random_call(L, dt, ct, bs, nb, n, counts, seed=3):
    """b200spmm_bsr on random data: returns (call(split) -> C tensor)"""
    g = torch.Generator(device=DEV).manual_seed(seed)
    off, col = R.pattern(nb, nb, counts, seed=seed)
    m = nb * bs
    V = torch.randn(len(col) * bs * bs, device=DEV, generator=g).to(dt)
    B = torch.randn(m, n, device=DEV, generator=g).to(dt)
    offd, cold = torch.tensor(off, dtype=torch.int32, device=DEV), torch.tensor(col, dtype=torch.int32, device=DEV)
    Cm = torch.zeros(m * n, dtype=ct, device=DEV)
    wsb = L.b200spmm_bsr_workspace_bytes(VT[dt], m, n, bs, len(col), 1)
    ws = torch.empty(max(wsb, 16), dtype=torch.uint8, device=DEV)
    one, zero = (C.c_double(1.0), C.c_double(0.0)) if dt == torch.float64 else (C.c_float(1.0), C.c_float(0.0))

    def call(stream, split=True):
        assert L.b200spmm_bsr(stream.cuda_stream, VT[dt], VT[ct], m, m, n, bs, len(col), offd.data_ptr(), cold.data_ptr(), V.data_ptr(), 0,
                              1, C.addressof(one), C.addressof(zero), 0, B.data_ptr(), n, 1, Cm.data_ptr(), n, 1, 1, 0, 0, 0, 0, 0,
                              ws.data_ptr() if split else None, wsb if split else 0) == 0
    return call, Cm


@pytest.mark.parametrize("dt,ct,bs", [(torch.float16, torch.float32, 16), (torch.bfloat16, torch.bfloat16, 64), (torch.float32, torch.float32, 8),
                                      (torch.float64, torch.float64, 4)])
def test_repeat_graph_replay_and_null_buffer_are_bit_identical(L, dt, ct, bs):
    call, Cm = random_call(L, dt, ct, bs, 24, 72, [3, 24, 5, 0, 7])          # a global block-row: the split walk cuts it
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
def test_parity_with_the_closed_library_on_random_data(L, dt, ct, order):
    """ours and the closed cusparseSpMM on the same buffers, both within the dot-product bound of fp64 (where it accepts the call)"""
    import scripts.spmm_bsr_bench as SB
    bs = 32
    off, col = SB.pattern("window", 16, seed=bs)
    row = SB.run_case(L, "window", 16 * bs, bs, 72, dt, ct, order, off, col)
    u = {torch.float16: 2.0 ** -11, torch.bfloat16: 2.0 ** -8, torch.float32: 2.0 ** -24, torch.float64: 2.0 ** -53}
    acc_u = 2.0 ** -53 if dt == torch.float64 else 2.0 ** -24
    kmax = 16 * bs
    tol = kmax * acc_u + 2 * u[ct]
    assert row["err_ours"] <= tol, row
    if "err_closed" in row:
        assert row["err_closed"] <= 4 * tol, row


# ------------------------------------------------------------------------------------------------ through the shim
@pytest.fixture(scope="module")
def cs():
    from cudalibrarysamples_b200 import cusparse_api
    return cusparse_api


def attempt(fn):
    """("ok", result) or ("status", the error) of a call that either library may refuse"""
    from cudalibrarysamples_b200 import cusparse_api
    try:
        return ("ok", fn())
    except cusparse_api.CuSparseError as e:
        return ("status", str(e))


def shim_spmm(cs, impl, dt, ct, bs, off, col, val, b, c0, batches=1, **kw):
    api = cs.Api(impl)
    m = (len(off) - 1) * bs
    arr = dict(off=torch.tensor(off, dtype=torch.int32, device=DEV), col=torch.tensor(col, dtype=torch.int32, device=DEV),
               val=torch.tensor(val, dtype=dt, device=DEV), bnnz=len(col) // batches if batches > 1 and kw.get("col_stride") != 0 else len(col))
    B = torch.tensor(b, dtype=dt, device=DEV).contiguous().view(-1)
    C0 = torch.tensor(c0, dtype=ct, device=DEV).contiguous().view(-1)
    return cs.spmm_bsr(api, m, b.shape[-2], b.shape[-1], bs, arr, B, C0, 1.0, 1.0, batches=batches, **kw).double().cpu().numpy()


@pytest.mark.parametrize("dt,ct", [(torch.float16, torch.float16), (torch.float16, torch.float32), (torch.bfloat16, torch.bfloat16),
                                   (torch.bfloat16, torch.float32)], ids=["f16", "f16-f32", "bf16", "bf16-f32"])
@pytest.mark.parametrize("bs,n,heads", [(64, 64, 1), (128, 128, 1), (16, 64, 16)])
def test_shim_runs_the_measured_class_natively(L, cs, dt, ct, bs, n, heads):
    """the attention layout at sequence length 4096 (bs 16: 16 heads in one batch): native through cusparseSpMM with nothing forwarded, exact, and equal to the
    closed library's result"""
    nb = 4096 // bs
    off, col = R.pattern(nb, nb, [1, 0, 3, 2, nb], seed=6)
    vals, bs_, cs_, exp = [], [], [], []
    for h in range(heads):
        val, b, c0 = R.values(nb * bs, nb * bs, n, len(col), bs, seed=7 + h)
        vals.append(val); bs_.append(b); cs_.append(c0)
        R.check_exact(nb * bs, nb * bs, bs, off, col, val, b, c0, 1.0, 1.0, KIND[ct])
        exp.append(R.reference(nb * bs, nb * bs, bs, off, col, val, b, c0, 1.0, 1.0))
    b200 = cs.Api("b200")
    b200.reset_stats()
    got = shim_spmm(cs, "b200", dt, ct, bs, off, col, np.concatenate(vals), np.stack(bs_), np.stack(cs_), batches=heads, col_stride=0)
    st = b200.stats()
    assert st["native"] == 1 and st["forwarded"] == 0, st
    assert np.array_equal(got, np.concatenate([e.ravel() for e in exp]))
    closed = attempt(lambda: shim_spmm(cs, "cusparse", dt, ct, bs, off, col, np.concatenate(vals), np.stack(bs_), np.stack(cs_),
                                       batches=heads, col_stride=0))
    assert closed[0] == "ok" and np.array_equal(closed[1], got)


def test_forwarded_kinds_are_counted(L, cs):
    """opA = T, CONJUGATE_TRANSPOSE, 64-bit indices, a mixed type, a non-default algorithm and a small fp32 class never run
    natively; they get the closed library's status or result"""
    b200 = cs.Api("b200")
    off, col, val, b, c0 = case(4, 4, 4, 8)

    def op_a(op):
        def f(impl):
            api = cs.Api(impl)
            h = api.cusparseCreate()
            arr = [torch.tensor(x, device=DEV) for x in (off, col)]
            A = api.cusparseCreateBsr(4, 4, len(col), 4, 4, arr[0].int(), arr[1].int(), torch.tensor(val, dtype=torch.float32, device=DEV))
            B = torch.tensor(b, dtype=torch.float32, device=DEV).contiguous()
            Cm = torch.tensor(c0, dtype=torch.float32, device=DEV).contiguous()
            mB, mC = api.cusparseCreateDnMat(16, 8, 8, B, ROW), api.cusparseCreateDnMat(16, 8, 8, Cm, ROW)
            try:
                size = api.cusparseSpMM_bufferSize(h, op, NT, 1.0, A, mB, 1.0, mC, 0)
                buf = torch.empty(max(size, 16), dtype=torch.uint8, device=DEV)
                api.cusparseSpMM(h, op, NT, 1.0, A, mB, 1.0, mC, 0, 0, buf)
                torch.cuda.synchronize()
            finally:
                api.cusparseDestroySpMat(A); api.cusparseDestroyDnMat(mB); api.cusparseDestroyDnMat(mC); api.cusparseDestroy(h)
            return Cm.double().cpu().numpy()
        return f

    def int64_call(impl):
        api = cs.Api(impl)
        arr = dict(off=torch.tensor(off, dtype=torch.int64, device=DEV), col=torch.tensor(col, dtype=torch.int64, device=DEV),
                   val=torch.tensor(val, dtype=torch.float32, device=DEV))
        return cs.spmm_bsr(api, 16, 16, 8, 4, arr, torch.tensor(b, dtype=torch.float32, device=DEV).view(-1),
                           torch.tensor(c0, dtype=torch.float32, device=DEV).view(-1), 1.0, 1.0).double().cpu().numpy()
    fns = (op_a(TR), op_a(2), int64_call,
           lambda impl: shim_spmm(cs, impl, torch.float32, torch.float64, 4, off, col, val, b, c0, compute=0),
           lambda impl: shim_spmm(cs, impl, torch.float32, torch.float32, 4, off, col, val, b, c0, alg=6),
           lambda impl: shim_spmm(cs, impl, torch.float32, torch.float32, 4, off, col, val, b, c0))
    for i, fn in enumerate(fns):
        got = {}
        for impl in ("b200", "cusparse"):
            b200.reset_stats()
            got[impl] = attempt(lambda: fn(impl))
            if impl == "b200":
                st = b200.stats()
                assert st["native"] == 0 and st["forwarded"] == (1 if got[impl][0] == "ok" else st["forwarded"]), (i, st)
        assert got["b200"][0] == got["cusparse"][0], (i, got)
        if got["b200"][0] == "ok":
            assert np.array_equal(got["b200"][1], got["cusparse"][1]), i


def test_status_parity_for_shape_mismatches(L, cs):
    """on a natively routed class: B with one row more than A has columns, and C with one row more than A"""
    bs, nb, n = 64, 64, 64
    off, col = R.pattern(nb, nb, [1, 2], seed=2)
    sts = {}
    for impl in ("b200", "cusparse"):
        for what in ("k", "m", "n"):
            api = cs.Api(impl)
            h = api.cusparseCreate()
            V = torch.zeros(len(col) * bs * bs, dtype=torch.float16, device=DEV)
            B = torch.zeros((nb * bs + 1) * (n + 1), dtype=torch.float16, device=DEV)
            Cm = torch.zeros((nb * bs + 1) * (n + 1), dtype=torch.float16, device=DEV)
            A = api.cusparseCreateBsr(nb, nb, len(col), bs, bs, torch.tensor(off, dtype=torch.int32, device=DEV),
                                      torch.tensor(col, dtype=torch.int32, device=DEV), V)
            mB = api.cusparseCreateDnMat(nb * bs + (what == "k"), n, n, B, ROW)
            mC = api.cusparseCreateDnMat(nb * bs + (what == "m"), n + (what == "n"), n + (what == "n"), Cm, ROW)

            def call():
                size = api.cusparseSpMM_bufferSize(h, NT, NT, 1.0, A, mB, 0.0, mC, 0)
                buf = torch.empty(max(size, 16), dtype=torch.uint8, device=DEV)
                api.cusparseSpMM_preprocess(h, NT, NT, 1.0, A, mB, 0.0, mC, 0, 0, buf)
                api.cusparseSpMM(h, NT, NT, 1.0, A, mB, 0.0, mC, 0, 0, buf)
                torch.cuda.synchronize()
            sts[(impl, what)] = attempt(call)[0]
            api.cusparseDestroyDnMat(mB); api.cusparseDestroyDnMat(mC); api.cusparseDestroySpMat(A); api.cusparseDestroy(h)
    for what in ("k", "m", "n"):
        assert sts[("b200", what)] == sts[("cusparse", what)], sts


def test_block_sparse_attention_head_end_to_end(L, cs):
    """S = Q . K^T on the pattern (cusparseSDDMM, BSR), P = softmax over each row's stored entries (torch), O = P . V (cusparseSpMM,
    BSR): both sparse calls native, O equal to dense masked attention in fp32"""
    import scripts.sddmm_bsr_bench as SB
    bs, seq, d = 64, 4096, 64
    nb = seq // bs
    off, col = SB.pattern("window", nb, seed=1)
    g = torch.Generator(device=DEV).manual_seed(0)
    Q, K, V = [(torch.randn(seq, d, device=DEV, generator=g) * 0.5).half() for _ in range(3)]
    api = cs.Api("b200")
    api.reset_stats()
    arr = dict(off=torch.tensor(off, dtype=torch.int32, device=DEV), col=torch.tensor(col, dtype=torch.int32, device=DEV),
               val=torch.zeros(len(col) * bs * bs, dtype=torch.float32, device=DEV))
    S = cs.sddmm_bsr(api, seq, seq, d, bs, Q, K, arr, 1.0 / d ** 0.5, 0.0, opB=TR)          # fp32 scores
    st = api.stats()
    assert st["native"] == 1 and st["forwarded"] == 0, st
    rows = torch.repeat_interleave(torch.arange(nb, device=DEV), torch.diff(arr["off"]).long())
    Sb = S.view(-1, bs, bs)                                               # block e: rows of block-row rows[e], row-major
    Sr = torch.full((nb, bs, nb * bs), float("-inf"), device=DEV)        # each block-row's scores on its stored columns
    cidx = arr["col"].long()[:, None] * bs + torch.arange(bs, device=DEV)[None, :]
    Sr[rows[:, None, None], torch.arange(bs, device=DEV)[None, :, None], cidx[:, None, :]] = Sb
    Pr = torch.softmax(Sr, dim=-1)
    P = Pr[rows[:, None, None], torch.arange(bs, device=DEV)[None, :, None], cidx[:, None, :]].half().contiguous().view(-1)
    O = torch.zeros(seq * d, dtype=torch.float32, device=DEV)
    pa = dict(off=arr["off"], col=arr["col"], val=P)
    api.reset_stats()
    cs.spmm_bsr(api, seq, seq, d, bs, pa, V.contiguous().view(-1), O, 1.0, 0.0)
    st = api.stats()
    assert st["native"] == 1 and st["forwarded"] == 0, st
    mask = torch.zeros(seq, seq, dtype=torch.bool, device=DEV)
    mask.view(nb, bs, nb, bs)[rows, :, arr["col"].long(), :] = True
    dense = (Q.float() @ K.float().T) / d ** 0.5
    dense = dense.masked_fill(~mask, float("-inf"))
    ref = torch.softmax(dense, dim=-1) @ V.float()
    err = (O.view(seq, d) - ref).abs().max().item()
    assert err < 2e-3, err
