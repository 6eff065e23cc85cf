"""GPU: the half-precision CSR SpMV (spmv_csr16.cu) bit for bit against the int64 reference on integer data over every type pair,
index base, scalar placement and row-length edge; bit for bit against the fp32 restatement of its summation on random data; both
walks, every kind of unusable buffer, repeats and graph replays bit-identical; NaN guards; parity with the closed library; and the
shim's routing and counting."""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import spmv_csr16_ref as R

pytestmark = pytest.mark.gpu

DEV = "cuda"
VT = {torch.float32: 0, torch.float16: 2, torch.bfloat16: 14}
KIND = {torch.float32: "f32", torch.float16: "f16", torch.bfloat16: "bf16"}
TYPES = [(torch.float16, torch.float16), (torch.float16, torch.float32), (torch.bfloat16, torch.bfloat16), (torch.bfloat16, torch.float32)]
IDS = ["f16-f16", "f16-f32", "bf16-bf16", "bf16-f32"]


@pytest.fixture(scope="module")
def L():
    from cudalibrarysamples_b200 import lib
    return lib.shim()


def dev(a, dtype, shift=0):
    """a device copy of a starting `shift` elements into its allocation; returns (allocation, pointer)"""
    t = torch.zeros(len(a) + shift + 1, dtype=dtype)
    if shift:
        t[:shift] = 7
    t[shift:shift + len(a)] = torch.from_numpy(np.asarray(a, np.float64 if dtype.is_floating_point else np.int64)).to(dtype)
    d = t.to(DEV)
    return d, d.data_ptr() + shift * d.element_size()


def run(L, dt, yt, off, col, val, x, y0=None, alpha=1.0, beta=0.0, base=0, on_device=False, ws="full", shift=0, cols=None):
    """one b200spmv_csr16 call; y is NaN where beta == 0.  ws: "full", None, "misaligned" or "small".  Returns y as float64 numpy."""
    rows = len(off) - 1
    cols = len(x) if cols is None else cols
    nnz = len(col)
    offd, po = dev(off, torch.int32)
    cold, pc = dev(col, torch.int32, shift)
    vald, pv = dev(val, dt, shift)
    xd, px = dev(x, dt, shift)
    yinit = np.full(rows, np.nan) if beta == 0 or y0 is None else np.asarray(y0, np.float64)
    yd, py = dev(yinit, yt, shift)
    if on_device:
        keep = (torch.tensor([alpha], dtype=torch.float32, device=DEV), torch.tensor([beta], dtype=torch.float32, device=DEV))
        pa, pb = keep[0].data_ptr(), keep[1].data_ptr()
    else:
        keep = (C.c_float(alpha), C.c_float(beta))
        pa, pb = C.addressof(keep[0]), C.addressof(keep[1])
    need = L.b200spmv_csr16_workspace_bytes(rows, nnz)
    buf = torch.full((need + 64,), 0x7F, dtype=torch.uint8, device=DEV)
    wp, wb = {"full": (buf.data_ptr(), need), None: (None, 0), "misaligned": (buf.data_ptr() + 4, need),
              "small": (buf.data_ptr(), max(need - 4, 0))}[ws]
    rc = L.b200spmv_csr16(torch.cuda.current_stream().cuda_stream, VT[dt], VT[yt], rows, cols, nnz, po, pc, pv, base, pa, pb,
                          int(on_device), px, py, wp, wb)
    torch.cuda.synchronize()
    assert rc == 0, rc
    return yd[shift:shift + rows].double().cpu().numpy()


def check(L, dt, yt, off, col, val, x, y0, alpha=1.0, beta=0.0, base=0, **kw):
    ref = R.reference_int(off, col, val, x, y0, alpha, beta, KIND[yt], base)
    for ws in ("full", None):
        got = run(L, dt, yt, off, col, val, x, y0, alpha, beta, base, ws=ws, **kw)
        assert np.array_equal(got, ref), (dt, yt, ws, kw, np.nanmax(np.abs(got - ref)), np.flatnonzero(got != ref)[:10])


def edge_lengths(E):
    return [0, 1, E - 1, E, E + 1, 0, 2 * E - 1, 2 * E + 1, 3, E, 0, 2 * E - 1, 2 * E, 2 * E + 1, 5, 0, 0, 1]


def sparse_x(k, seed, density):
    rng = np.random.default_rng(seed)
    return np.where(rng.random(k) < density, rng.choice([-1, 1], k), 0)


@pytest.mark.parametrize("dt,yt", TYPES, ids=IDS)
@pytest.mark.parametrize("base", [0, 1])
def test_exact_on_integer_data(L, dt, yt, base):
    E = R.params(L)["chunk"]
    k = 3 * E
    off, col = R.pattern(edge_lengths(E), k, seed=1, base=base)
    rng = np.random.default_rng(2)
    val = rng.choice([-1, 1], len(col))
    x = sparse_x(k, 3, 0.3 if yt == torch.bfloat16 else 1.0)
    y0 = 2 * rng.integers(-3, 4, len(off) - 1)
    for alpha, beta, on_device in ((1.0, 0.0, False), (2.0 if yt != torch.bfloat16 else 1.0, 0.5, False), (-1.0, 0.0, True),
                                   (-1.0, -2.0, True), (1.0, 1.0, False)):
        check(L, dt, yt, off, col, val, x, y0, alpha, beta, base, on_device=on_device)


@pytest.mark.parametrize("dt,yt", TYPES, ids=IDS)
def test_one_row_of_a_hundred_thousand_entries(L, dt, yt):
    """a hub row spread over ~400 chunks between short rows: exact, both walks"""
    k = 120000
    off, col = R.pattern([3, 0, 100000, 7, 0, 1, 2 * R.params(L)["chunk"] + 1], k, seed=5)
    rng = np.random.default_rng(6)
    val = rng.choice([-1, 1], len(col))
    x = sparse_x(k, 7, 0.002 if yt == torch.bfloat16 else 0.015)
    check(L, dt, yt, off, col, val, x, None)
    check(L, dt, yt, off, col, val, x, 2 * rng.integers(-3, 4, len(off) - 1), 1.0, 1.0)


@pytest.mark.parametrize("dt,yt", TYPES, ids=IDS)
def test_degenerate_shapes(L, dt, yt):
    # rows = 0: nothing happens
    one, zero = C.c_float(1.0), C.c_float(0.0)
    assert L.b200spmv_csr16(None, VT[dt], VT[yt], 0, 5, 0, None, None, None, 0, C.addressof(one), C.addressof(zero), 0, None, None, None,
                            0) == 0
    # nnz = 0: y = beta * y, and NaN-free under beta = 0
    y0 = np.array([2.0, -4.0, 6.0])
    for beta in (0.0, 0.5):
        got = run(L, dt, yt, np.zeros(4, np.int64), np.zeros(0, np.int64), np.zeros(0), np.ones(2), y0, 1.0, beta)
        assert np.array_equal(got, beta * y0), (beta, got)
    # 1 x 1
    check(L, dt, yt, np.array([0, 1]), np.array([0]), np.array([-1]), np.array([1]), np.array([2]), 2.0, 1.0)
    check(L, dt, yt, np.array([1, 2]), np.array([1]), np.array([1]), np.array([-1]), None, base=1)
    # all rows empty, many of them (one chunk owns them all)
    check(L, dt, yt, np.zeros(5001, np.int64), np.zeros(0, np.int64), np.zeros(0), np.ones(3), 2 * np.ones(5000), 1.0, -1.0)


@pytest.mark.parametrize("dt,yt", TYPES, ids=IDS)
def test_views_misaligned_by_one_element(L, dt, yt):
    E = R.params(L)["chunk"]
    off, col = R.pattern(edge_lengths(E), 3 * E, seed=8)
    rng = np.random.default_rng(9)
    val = rng.choice([-1, 1], len(col))
    x = sparse_x(3 * E, 10, 0.3)
    _, pc = dev(col, torch.int32, 1)
    _, pv = dev(val, dt, 1)
    assert L.b200spmv_csr16_path(pc, pv) == 1
    _, pc0 = dev(col, torch.int32)
    _, pv0 = dev(val, dt)
    assert L.b200spmv_csr16_path(pc0, pv0) == 2
    check(L, dt, yt, off, col, val, x, 2 * rng.integers(-3, 4, len(off) - 1), 1.0, 1.0, shift=1)
    check(L, dt, yt, off, col, val, x, None, shift=1)


def random_case(dt, lengths, k, seed):
    off, col = R.pattern(lengths, k, seed)
    g = torch.Generator().manual_seed(seed)
    # magnitudes from 2^-24 to 2: every product is a normal fp32 number, for bf16 too
    val = (torch.rand(len(col), generator=g) * 2 - 1).to(dt).double().numpy()
    x = (torch.rand(k, generator=g) * 4 - 2).to(dt).double().numpy()
    return off, col, val, x


@pytest.mark.parametrize("dt,yt", TYPES, ids=IDS)
def test_bit_identical_to_the_fp32_restatement_on_random_data(L, dt, yt):
    P = R.params(L)
    E = P["chunk"]
    for lengths, k in ((edge_lengths(E) * 3, 4 * E), ([5, 40 * E + 17, 0, 2, E + 1, 9] * 2, 50 * E), (list(range(0, 300)) * 2, 2000)):
        off, col, val, x = random_case(dt, lengths, k, seed=len(lengths))
        want = R.round_to(R.accumulate_f32(off, col, val, x, E, P["run"]), KIND[yt])
        for ws in ("full", None):
            got = run(L, dt, yt, off, col, val, x, ws=ws)
            bad = np.flatnonzero(got.view(np.int64) != want.view(np.int64))
            assert not len(bad), (ws, bad[:10], got[bad[:5]], want[bad[:5]])


@pytest.mark.parametrize("dt,yt", [(torch.float16, torch.float32), (torch.bfloat16, torch.bfloat16)], ids=["f16-f32", "bf16"])
def test_walks_buffers_repeats_and_graph_replays_are_bit_identical(L, dt, yt):
    E = R.params(L)["chunk"]
    lengths = [3, 5000, 0, 700, 1, 1300, E, E + 1] * 50
    off, col, val, x = random_case(dt, lengths, 8000, seed=11)
    rows, nnz = len(lengths), len(col)
    first = run(L, dt, yt, off, col, val, x)
    assert np.isfinite(first).all()
    for ws in ("full", None, "misaligned", "small", "full"):
        assert np.array_equal(run(L, dt, yt, off, col, val, x, ws=ws), first), ws
    offd, cold = torch.tensor(off, dtype=torch.int32, device=DEV), torch.tensor(col, dtype=torch.int32, device=DEV)
    vald, xd = torch.tensor(val, dtype=dt, device=DEV), torch.tensor(x, dtype=dt, device=DEV)
    yd = torch.full((rows,), float("nan"), dtype=yt, device=DEV)
    wsb = L.b200spmv_csr16_workspace_bytes(rows, nnz)
    ws = torch.full((wsb,), 0x7F, dtype=torch.uint8, device=DEV)
    one, zero = C.c_float(1.0), C.c_float(0.0)
    s = torch.cuda.Stream()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph, stream=s):
        assert L.b200spmv_csr16(s.cuda_stream, VT[dt], VT[yt], rows, 8000, nnz, offd.data_ptr(), cold.data_ptr(), vald.data_ptr(), 0,
                                C.addressof(one), C.addressof(zero), 0, xd.data_ptr(), yd.data_ptr(), ws.data_ptr(), wsb) == 0
    for _ in range(3):
        yd.fill_(float("nan"))
        graph.replay()
        torch.cuda.synchronize()
        assert np.array_equal(yd.double().cpu().numpy(), first)


@pytest.mark.parametrize("dt", [torch.float16, torch.bfloat16])
def test_nan_guards(L, dt):
    """NaN in x entries no row stores and in y under beta = 0 never reaches y; NaN in x[0] reaches exactly the rows storing column 0"""
    E = R.params(L)["chunk"]
    lengths = [4, 0, E + 3, 6, 1, 2 * E + 1, 0, 3]
    off, col = R.pattern(lengths, 3 * E, seed=12)
    col = col + 1                                                   # columns 1 .. 3E; 3E + 1 .. 3E + 9 are never stored
    rng = np.random.default_rng(13)
    val = rng.choice([-1, 1], len(col))
    x = np.r_[sparse_x(3 * E + 1, 14, 0.3), np.full(9, np.nan)]
    x[0] = 0
    ref = R.reference_int(off, col, val, np.nan_to_num(x), None, 1.0, 0.0, "f32")
    for ws in ("full", None):
        assert np.array_equal(run(L, dt, torch.float32, off, col, val, x, ws=ws), ref), ws
    col0 = col.copy()
    col0[off[0]] = col0[off[2] + E + 1] = col0[off[5]] = 0          # column 0 in rows 0, 2 (past its first E entries) and 5
    x[0] = np.nan
    stores0 = np.isin(np.arange(len(lengths)), [0, 2, 5])
    for ws in ("full", None):
        got = run(L, dt, torch.float32, off, col0, val, x, ws=ws)
        assert (np.isnan(got) == stores0).all(), (ws, got)


@pytest.mark.parametrize("dt,yt", TYPES, ids=IDS)
@pytest.mark.parametrize("which", ["rmat", "stencil"])
def test_parity_with_the_closed_library(L, dt, yt, which):
    """ours and the closed cusparseSpMV on the same buffers: both within the fp32 dot-product bound plus one rounding to y's type,
    relative to sum_k |a_rk| |x_k|"""
    import scripts.spmv_csr16_bench as SB
    from cudalibrarysamples_b200 import workloads as W
    if which == "rmat":
        m = 1 << 16
        off, col, val = W.rmat_csr(m, avg_nnz=16, seed=3, val_seed=4, dtype=torch.float32)
    else:
        off, col, val = W.stencil5_csr(512)
        m = 512 * 512
    row = SB.run_case(which, m, m, off.int(), col.int(), val.float(), dt, yt)
    u = {torch.float16: 2.0 ** -11, torch.bfloat16: 2.0 ** -8, torch.float32: 2.0 ** -24}
    kmax = int((off[1:] - off[:-1]).max())
    tol = kmax * 2.0 ** -24 + u[yt]
    assert row["err_ours"] <= tol, row
    assert row["err_closed"] <= 4 * tol, row


# ------------------------------------------------------------------------------------------------ through the shim
def shim_case(m, per, dt, seed=1):
    g = torch.Generator(device=DEV).manual_seed(seed)
    lengths = torch.full((m,), per, dtype=torch.int32, device=DEV)
    lengths[7], lengths[8] = 3000, 0                                 # one row crossing chunks, one empty row
    off = torch.zeros(m + 1, dtype=torch.int32, device=DEV)
    off[1:] = torch.cumsum(lengths, 0)
    nnz = int(off[-1])
    col = torch.randint(0, m, (nnz,), device=DEV, generator=g, dtype=torch.int32)
    rows = torch.repeat_interleave(torch.arange(m, device=DEV), lengths.long())
    col = col[torch.argsort(rows.long() * m + col.long())].contiguous()
    val = (torch.rand(nnz, device=DEV, generator=g) * 2 - 1).to(dt)
    x = (torch.rand(m, device=DEV, generator=g) * 2 - 1).to(dt)
    return dict(off=off, col=col, val=val), x


U = {torch.float16: 2.0 ** -11, torch.bfloat16: 2.0 ** -8, torch.float32: 2.0 ** -24}


def rel_err(y, yc, arrays, x):
    """largest |y - yc| relative to sum_k |a_rk| |x_k|"""
    m = y.numel()
    A = torch.sparse_csr_tensor(arrays["off"], arrays["col"], arrays["val"].float().abs(), (m, x.numel()))
    bound = (A @ x.float().abs().unsqueeze(1)).squeeze(1).double()
    return ((yc.double() - y.double()).abs() / (bound + 1e-30)).max().item()


def native_shape(dt, yt):
    from scripts.spmv_csr16_bench import NATIVE
    for m, per in ((1 << 20, 16), (2 << 20, 16), (1 << 20, 5), (4 << 20, 8), (16 << 20, 5), (10 << 20, 16)):
        if eval(NATIVE)(VT[dt], VT[yt], m, m, m * per + 3000 - per * 2):
            return m, per
    return None


@pytest.mark.parametrize("dt,yt", TYPES, ids=IDS)
def test_shim_serves_a_routed_shape_natively(L, dt, yt):
    """bufferSize >= the closed library's, preprocess succeeds, the call is counted native with nothing forwarded, the log names the
    kernel, and y equals b200spmv_csr16 with the same buffer; then the same call captured in a CUDA graph"""
    from cudalibrarysamples_b200 import cusparse_api as cs
    shape = native_shape(dt, yt)
    if shape is None:
        pytest.skip("the route serves no measured shape of this type pair")
    m, per = shape
    arrays, x = shim_case(m, per, dt)
    nnz = arrays["col"].numel()
    closed = cs.SpMVOperator(cs.Api("cusparse"), "csr", m, m, arrays, y_dtype=yt, compute_dtype=torch.float32)
    yc = torch.zeros(m, dtype=yt, device=DEV)
    closed(x, yc)
    torch.cuda.synchronize()
    api = cs.Api("b200")
    api.reset_stats()
    op = cs.SpMVOperator(api, "csr", m, m, arrays, y_dtype=yt, compute_dtype=torch.float32)
    assert op.buffer_bytes >= closed.buffer_bytes and op.buffer_bytes >= L.b200spmv_csr16_workspace_bytes(m, nnz)
    assert L.b200spmv_route(1, 0, 0, 2, 2, VT[dt], VT[dt], VT[yt], 0, m, m, nnz) == 3
    assert L.b200spmv_csr16_route(op.mat, op.vecX, op.vecY, 0, 0, 0) == 3
    y = torch.full((m,), float("nan"), dtype=yt, device=DEV)
    op(x, y)
    torch.cuda.synchronize()
    st = api.stats()
    assert st["native"] == 1 and st["forwarded"] == 0 and st["analyze"] == 0, st
    assert "spmv_csr16_chunk_kernel" in api.last_csr_kernel()
    direct = torch.full_like(y, float("nan"))
    one, zero = C.c_float(1.0), C.c_float(0.0)
    assert L.b200spmv_csr16(torch.cuda.current_stream().cuda_stream, VT[dt], VT[yt], m, m, nnz, arrays["off"].data_ptr(),
                            arrays["col"].data_ptr(), arrays["val"].data_ptr(), 0, C.addressof(one), C.addressof(zero), 0, x.data_ptr(),
                            direct.data_ptr(), op.buffer.data_ptr(), op.buffer_bytes) == 0
    torch.cuda.synchronize()
    assert torch.equal(y, direct)
    assert rel_err(y, yc, arrays, x) < 4 * (U[yt] + 3000 * 2.0 ** -24)
    # graph capture of the shim call
    s = torch.cuda.Stream()
    api.cusparseSetStream(op.handle, s.cuda_stream)
    call = op.prebuilt(x, y)
    with torch.cuda.stream(s):
        call()
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph, stream=s):
        call()
    for _ in range(2):
        y.fill_(float("nan"))
        graph.replay()
        torch.cuda.synchronize()
        assert torch.equal(y, direct)
    op.close()
    closed.close()


@pytest.mark.parametrize("dt,yt", TYPES, ids=IDS)
def test_forwarded_16bit_calls_are_counted(L, dt, yt):
    """a 16-bit CSR SpMV outside the routed shapes goes to the closed library, counted as forwarded, with its result"""
    from cudalibrarysamples_b200 import cusparse_api as cs
    m = 4096
    arrays, x = shim_case(m, 8, dt, seed=2)
    assert L.b200spmv_route(1, 0, 0, 2, 2, VT[dt], VT[dt], VT[yt], 0, m, m, arrays["col"].numel()) == 0
    api = cs.Api("b200")
    api.reset_stats()
    op = cs.SpMVOperator(api, "csr", m, m, arrays, y_dtype=yt, compute_dtype=torch.float32)
    y = torch.zeros(m, dtype=yt, device=DEV)
    op(x, y)
    torch.cuda.synchronize()
    st = api.stats()
    assert st["native"] == 0 and st["forwarded"] == 1, st
    closed = cs.SpMVOperator(cs.Api("cusparse"), "csr", m, m, arrays, y_dtype=yt, compute_dtype=torch.float32)
    yc = torch.zeros(m, dtype=yt, device=DEV)
    closed(x, yc)
    torch.cuda.synchronize()
    assert rel_err(y, yc, arrays, x) < 4 * (U[yt] + 3000 * 2.0 ** -24)
    op.close()
    closed.close()
