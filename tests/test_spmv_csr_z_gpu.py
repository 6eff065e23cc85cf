"""GPU: the double-complex CSR SpMV (spmv_csr_z.cu) bit for bit against the exact Gaussian-integer reference for opA N / T / C over
index bases, scalar placement, beta = 0 on a NaN-filled y, empty rows, a 100 000-entry row and the chunk edges; opA = N bit for bit
against the fp64 restatement of its arithmetic on random data, identical across both walks, repeats and graph replays; T / C within
tolerance of scipy; parity with the closed library; and the shim's routing and counting."""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import spmv_csr_z_ref as R

pytestmark = pytest.mark.gpu

DEV = "cuda"
OPS = {"N": 0, "T": 1, "C": 2}
NAN = complex(float("nan"), float("nan"))


@pytest.fixture(scope="module")
def L():
    from cudalibrarysamples_b200 import lib
    return lib.shim()


def cplx(a, dtype=torch.complex128):
    return torch.from_numpy(np.asarray(a, np.complex128)).to(DEV)


def run(L, op, off, col, val, x, rows, cols, y0=None, alpha=1, beta=0, base=0, on_device=False, ws="full"):
    """one b200spmv_csr_z call; y starts as NaN where beta == 0.  ws: "full", None, "misaligned" or "small".  Returns y (numpy)."""
    nnz = len(col)
    ny = rows if op == "N" else cols
    offd = torch.tensor(np.asarray(off, np.int64), dtype=torch.int32, device=DEV)
    cold = torch.tensor(np.asarray(col, np.int64), dtype=torch.int32, device=DEV) if nnz else torch.zeros(1, dtype=torch.int32, device=DEV)
    vald = cplx(val) if nnz else torch.zeros(1, dtype=torch.complex128, device=DEV)
    xd = cplx(x) if len(x) else torch.zeros(1, dtype=torch.complex128, device=DEV)
    yd = cplx(np.full(ny, NAN) if beta == 0 or y0 is None else y0) if ny else torch.zeros(1, dtype=torch.complex128, device=DEV)
    if on_device:
        keep = (torch.tensor([alpha], dtype=torch.complex128, device=DEV), torch.tensor([beta], dtype=torch.complex128, device=DEV))
        pa, pb = keep[0].data_ptr(), keep[1].data_ptr()
    else:
        from cudalibrarysamples_b200.cusparse_api import CDoubleComplex
        keep = (CDoubleComplex(alpha), CDoubleComplex(beta))
        pa, pb = C.addressof(keep[0]), C.addressof(keep[1])
    need = L.b200spmv_csr_z_workspace_bytes(rows, nnz)
    buf = torch.full((need + 64,), 0x7F, dtype=torch.uint8, device=DEV)
    wp, wb = {"full": (buf.data_ptr(), need), None: (None, 0), "misaligned": (buf.data_ptr() + 8, need),
              "small": (buf.data_ptr(), max(need - 16, 0))}[ws]
    rc = L.b200spmv_csr_z(torch.cuda.current_stream().cuda_stream, OPS[op], rows, cols, nnz, offd.data_ptr(), cold.data_ptr(),
                          vald.data_ptr(), base, pa, pb, int(on_device), xd.data_ptr(), yd.data_ptr(), wp, wb)
    torch.cuda.synchronize()
    assert rc == 0, rc
    return yd[:ny].cpu().numpy()


def check(L, op, off, col, val, x, rows, cols, y0, alpha=1, beta=0, base=0, **kw):
    ref = R.reference_int(off, col, val, x, y0, alpha, beta, op, base, cols=cols)
    for ws in (("full", None) if op == "N" else ("full",)):
        got = run(L, op, off, col, val, x, rows, cols, y0, alpha, beta, base, ws=ws, **kw)
        assert np.array_equal(got, ref), (op, ws, kw, np.flatnonzero(got != ref)[:10])


def edge_lengths(E):
    return [0, 1, E - 1, E, E + 1, 0, 2 * E - 1, 2 * E + 1, 3, E, 0, 2 * E - 1, 2 * E, 2 * E + 1, 5, 0, 0, 1]


@pytest.mark.parametrize("op", ["N", "T", "C"])
@pytest.mark.parametrize("base", [0, 1])
def test_exact_on_gaussian_integers(L, op, base):
    E = R.params(L)["chunk"]
    lengths = edge_lengths(E)
    rows, k = len(lengths), 3 * E
    off, col = R.pattern(lengths, k, seed=1, base=base)
    val, xn, yn = R.values(rows, k, len(col), seed=2)
    x, y0 = (xn, yn) if op == "N" else (R.values(rows, 0, 0, seed=3)[2], R.values(0, k, 0, seed=4)[1])   # x[rows], y[k]
    for alpha, beta, on_device in ((1, 0, False), (2 - 1j, 2j, False), (-1j, 0, True), (1 + 1j, -2, True), (1, 1, False)):
        check(L, op, off, col, val, x, rows, k, y0, alpha, beta, base, on_device=on_device)


@pytest.mark.parametrize("op", ["N", "T", "C"])
def test_one_row_of_a_hundred_thousand_entries(L, op):
    """a hub row spread over ~400 chunks between short rows: exact, both walks"""
    k = 120000
    lengths = [3, 0, 100000, 7, 0, 1, 2 * R.params(L)["chunk"] + 1]
    off, col = R.pattern(lengths, k, seed=5)
    rows = len(lengths)
    val, xn, yn = R.values(rows, k, len(col), seed=6, lo=-1, hi=1)
    x, y0 = (xn, yn) if op == "N" else (yn, xn)
    check(L, op, off, col, val, x, rows, k, None)
    check(L, op, off, col, val, x, rows, k, y0, 1j, 1 - 1j)


@pytest.mark.parametrize("op", ["N", "T"])
def test_chunk_edges_and_degenerate_shapes(L, op):
    E = R.params(L)["chunk"]
    for n in (E - 1, E, E + 1):                     # one row of E - 1 / E / E + 1 entries, and as many rows of one entry
        for lengths in ([n], [1] * n, [0, n, 0]):
            off, col = R.pattern(lengths, n + 1, seed=n)
            rows = len(lengths)
            val, xn, yn = R.values(rows, n + 1, len(col), seed=n + 1)
            x, y0 = (xn, yn) if op == "N" else (yn, xn)
            check(L, op, off, col, val, x, rows, n + 1, y0, 1 + 1j, -1)
    # rows = 0 (N) / cols = 0 (T): nothing happens
    from cudalibrarysamples_b200.cusparse_api import CDoubleComplex
    one, zero = CDoubleComplex(1), CDoubleComplex(0)
    assert L.b200spmv_csr_z(None, 0, 0, 5, 0, None, None, None, 0, C.addressof(one), C.addressof(zero), 0, None, None, None, 0) == 0
    assert L.b200spmv_csr_z(None, 1, 5, 0, 0, None, None, None, 0, C.addressof(one), C.addressof(zero), 0, None, None, None, 0) == 0
    # nnz = 0: y = beta * y, and NaN-free under beta = 0
    y0 = np.array([2 + 1j, -4j, 6])
    for beta in (0, 2 - 1j):
        got = run(L, op, np.zeros(4, np.int64), [], [], np.ones(3 if op == "N" else 3), 3, 3, y0, 1, beta)
        assert np.array_equal(got, R.reference_int(np.zeros(4, np.int64), [], [], np.ones(3), y0, 1, beta, op, cols=3)), (beta, got)
    # all rows empty, many of them (one chunk owns them all)
    if op == "N":
        check(L, op, np.zeros(5001, np.int64), [], [], np.ones(3), 5000, 3, 2 * np.ones(5000), 1, -1j)


def test_misaligned_complex_arrays_are_rejected(L):
    from cudalibrarysamples_b200.cusparse_api import CDoubleComplex
    one = CDoubleComplex(1)
    off = torch.tensor([0, 1], dtype=torch.int32, device=DEV)
    col = torch.zeros(1, dtype=torch.int32, device=DEV)
    buf = torch.zeros(8, dtype=torch.complex128, device=DEV)
    p = buf.data_ptr()
    for op in (0, 1, 2):
        def call(v=p, x=p + 16, y=p + 32):
            return L.b200spmv_csr_z(None, op, 1, 1, 1, off.data_ptr(), col.data_ptr(), v, 0, C.addressof(one), C.addressof(one), 0, x, y,
                                    None, 0)
        assert call(v=p + 8) == -1 and call(x=p + 24) == -1 and call(y=p + 40) == -1
        assert call() == 0
    torch.cuda.synchronize()


def random_case(lengths, k, seed):
    off, col = R.pattern(lengths, k, seed)
    rng = np.random.default_rng(seed)
    val = rng.standard_normal(len(col)) + 1j * rng.standard_normal(len(col))
    x = rng.standard_normal(k) + 1j * rng.standard_normal(k)
    y0 = rng.standard_normal(len(lengths)) + 1j * rng.standard_normal(len(lengths))
    return off, col, val, x, y0


def test_n_is_bit_identical_to_the_restatement_on_random_data(L):
    P = R.params(L)
    E = P["chunk"]
    for lengths, k, alpha, beta in ((edge_lengths(E) * 2, 4 * E, 1, 0), ([5, 20 * E + 17, 0, 2, E + 1, 9], 30 * E, 0.3 - 1.7j, 0),
                                    (list(range(0, 120)) * 2, 2000, -0.5 + 0.25j, 1.5 + 0.5j)):
        off, col, val, x, y0 = random_case(lengths, k, seed=len(lengths))
        want = R.restate_n(off, col, val, x, y0, alpha, beta, E, P["run"])
        for ws in ("full", None):
            got = run(L, "N", off, col, val, x, len(lengths), k, y0, alpha, beta, ws=ws)
            bad = np.flatnonzero(got.view(np.int64) != want.view(np.int64))
            assert not len(bad), (ws, bad[:10], got.view(np.complex128)[bad[:5] // 2], want[bad[:5] // 2])


def test_walks_buffers_repeats_and_graph_replays_are_bit_identical(L):
    from cudalibrarysamples_b200.cusparse_api import CDoubleComplex
    E = R.params(L)["chunk"]
    lengths = [3, 5000, 0, 700, 1, 1300, E, E + 1] * 30
    off, col, val, x, _ = random_case(lengths, 8000, seed=11)
    rows, nnz = len(lengths), len(col)
    first = run(L, "N", off, col, val, x, rows, 8000, alpha=0.5 + 2j)
    assert np.isfinite(first).all()
    for ws in ("full", None, "misaligned", "small", "full"):
        assert np.array_equal(run(L, "N", off, col, val, x, rows, 8000, alpha=0.5 + 2j, ws=ws).view(np.int64), first.view(np.int64)), ws
    offd, cold = torch.tensor(off, dtype=torch.int32, device=DEV), torch.tensor(col, dtype=torch.int32, device=DEV)
    vald, xd = cplx(val), cplx(x)
    yd = torch.full((rows,), NAN, dtype=torch.complex128, device=DEV)
    wsb = L.b200spmv_csr_z_workspace_bytes(rows, nnz)
    ws = torch.full((wsb,), 0x7F, dtype=torch.uint8, device=DEV)
    a, z = CDoubleComplex(0.5 + 2j), CDoubleComplex(0)
    s = torch.cuda.Stream()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph, stream=s):
        assert L.b200spmv_csr_z(s.cuda_stream, 0, rows, 8000, nnz, offd.data_ptr(), cold.data_ptr(), vald.data_ptr(), 0, C.addressof(a),
                                C.addressof(z), 0, xd.data_ptr(), yd.data_ptr(), ws.data_ptr(), wsb) == 0
    for _ in range(3):
        yd.fill_(NAN)
        graph.replay()
        torch.cuda.synchronize()
        assert np.array_equal(yd.cpu().numpy().view(np.int64), first.view(np.int64))


@pytest.mark.parametrize("op", ["T", "C"])
def test_transposes_agree_with_scipy(L, op):
    import scipy.sparse as sp
    lengths = [3, 5000, 0, 700, 1, 1300, 17, 256] * 10
    k = 6000
    off, col, val, _, _ = random_case(lengths, k, seed=21)
    rng = np.random.default_rng(22)
    x = rng.standard_normal(len(lengths)) + 1j * rng.standard_normal(len(lengths))
    y0 = rng.standard_normal(k) + 1j * rng.standard_normal(k)
    A = sp.csr_matrix((val, col, off), shape=(len(lengths), k))
    At = A.T.conj() if op == "C" else A.T
    alpha, beta = 0.75 + 0.5j, 0.5 - 0.25j
    want = alpha * (At @ x) + beta * y0
    bound = abs(alpha) * (abs(At) @ np.abs(x)) + abs(beta) * np.abs(y0)
    got = run(L, op, off, col, val, x, len(lengths), k, y0, alpha, beta)
    kmax = int(np.bincount(col, minlength=k).max())
    assert (np.abs(got - want) <= (kmax + 4) * 2.0 ** -52 * 4 * bound + 1e-300).all()


@pytest.mark.parametrize("op", [0, 1, 2], ids=["N", "T", "C"])
@pytest.mark.parametrize("which", ["rmat", "stencil"])
def test_parity_with_the_closed_library(L, op, which):
    """ours and the closed cusparseSpMV on the same buffers: both within the fp64 dot-product bound of the fp64 reference"""
    import scripts.spmv_csr_z_bench as SB
    from cudalibrarysamples_b200 import workloads as W
    if which == "rmat":
        m = 1 << 16
        off, col, val = W.rmat_csr(m, avg_nnz=16, seed=3, val_seed=4, dtype=torch.float64)
    else:
        off, col, val = W.stencil5_csr(512)
        m = 512 * 512
    vals = torch.complex(val.double(), torch.rand(col.numel(), dtype=torch.float64, device=DEV) - 0.5)
    for beta in (0j, SB.BETA):
        row = SB.run_case(which, m, m, off.int(), col.int(), vals, op, beta)
        lens = (off[1:] - off[:-1]) if op == 0 else torch.bincount(col.long(), minlength=m)
        tol = (int(lens.max()) + 4) * 4 * 2.0 ** -52
        assert row["err_ours"] <= tol, row
        assert row["err_closed"] <= 4 * tol, row


# ------------------------------------------------------------------------------------------------ through the shim
def shim_case(m, per, seed=1):
    g = torch.Generator(device=DEV).manual_seed(seed)
    lengths = torch.full((m,), per, dtype=torch.int32, device=DEV)
    lengths[7], lengths[8] = 3000, 0                                 # one row crossing chunks, one empty row
    off = torch.zeros(m + 1, dtype=torch.int32, device=DEV)
    off[1:] = torch.cumsum(lengths, 0)
    nnz = int(off[-1])
    col = torch.randint(0, m, (nnz,), device=DEV, generator=g, dtype=torch.int32)
    rows = torch.repeat_interleave(torch.arange(m, device=DEV), lengths.long())
    col = col[torch.argsort(rows.long() * m + col.long())].contiguous()
    val = torch.complex(torch.rand(nnz, device=DEV, generator=g, dtype=torch.float64) - 0.5,
                        torch.rand(nnz, device=DEV, generator=g, dtype=torch.float64) - 0.5)
    x = torch.complex(torch.rand(m, device=DEV, generator=g, dtype=torch.float64) - 0.5,
                      torch.rand(m, device=DEV, generator=g, dtype=torch.float64) - 0.5)
    return dict(off=off, col=col, val=val), x


def rel_err(y, yc, arrays, x, op):
    m = y.numel()
    A = torch.sparse_csr_tensor(arrays["off"], arrays["col"], arrays["val"].abs(), (m, m)).to_dense() if m <= 8192 else None
    if A is None:
        bound = torch.ones(m, dtype=torch.float64, device=DEV) * float(arrays["val"].abs().max() * x.abs().max() * 3000)
    else:
        bound = (A.T if op else A) @ x.abs()
    return ((yc - y).abs() / (bound + 1e-30)).max().item()


def native_shape(op):
    from scripts.spmv_csr_z_bench import NATIVE
    for m, per in ((1 << 20, 16), (2 << 20, 16), (1 << 20, 5), (4 << 20, 7), (8 << 20, 5), (10 << 20, 16)):
        if eval(NATIVE)(op, m, m, m * per + 3000 - per * 2):
            return m, per
    return None


@pytest.mark.parametrize("op", [0, 1, 2], ids=["N", "T", "C"])
def test_shim_serves_a_routed_case_natively(L, op):
    """bufferSize >= the closed library's, preprocess succeeds, the call is counted native with nothing forwarded, the log names the
    kernel, and y equals b200spmv_csr_z's; for opA = N also the same call captured in a CUDA graph"""
    from cudalibrarysamples_b200 import cusparse_api as cs
    shape = native_shape(op)
    if shape is None:
        pytest.skip("the route serves no measured case of this opA")
    m, per = shape
    arrays, x = shim_case(m, per)
    nnz = arrays["col"].numel()
    closed = cs.SpMVOperator(cs.Api("cusparse"), "csr", m, m, arrays, op=op)
    yc = torch.zeros(m, dtype=torch.complex128, device=DEV)
    closed(x, yc, 1 - 1j)
    torch.cuda.synchronize()
    api = cs.Api("b200")
    api.reset_stats()
    o = cs.SpMVOperator(api, "csr", m, m, arrays, op=op)
    assert o.buffer_bytes >= closed.buffer_bytes and (op != 0 or o.buffer_bytes >= L.b200spmv_csr_z_workspace_bytes(m, nnz))
    assert L.b200spmv_route(1, op, 0, 2, 2, 5, 5, 5, 5, m, m, nnz) == 4
    assert L.b200spmv_csr16_route(o.mat, o.vecX, o.vecY, op, 5, 0) == 4
    y = torch.full((m,), NAN, dtype=torch.complex128, device=DEV) if op == 0 else torch.zeros(m, dtype=torch.complex128, device=DEV)
    o(x, y, 1 - 1j)
    torch.cuda.synchronize()
    st = api.stats()
    assert st["native"] == 1 and st["forwarded"] == 0 and st["analyze"] == 0, st
    assert "spmv_csrz_" in api.last_csr_kernel()
    assert rel_err(y, yc, arrays, x, op) < 3000 * 2.0 ** -48
    if op != 0:
        o.close()
        closed.close()
        return
    from cudalibrarysamples_b200.cusparse_api import CDoubleComplex
    direct = torch.full_like(y, NAN)
    a, z = CDoubleComplex(1 - 1j), CDoubleComplex(0)
    assert L.b200spmv_csr_z(torch.cuda.current_stream().cuda_stream, 0, m, m, nnz, arrays["off"].data_ptr(), arrays["col"].data_ptr(),
                            arrays["val"].data_ptr(), 0, C.addressof(a), C.addressof(z), 0, x.data_ptr(), direct.data_ptr(),
                            o.buffer.data_ptr(), o.buffer_bytes) == 0
    torch.cuda.synchronize()
    assert torch.equal(y, direct)
    s = torch.cuda.Stream()
    api.cusparseSetStream(o.handle, s.cuda_stream)
    call = o.prebuilt(x, y, 1 - 1j)
    with torch.cuda.stream(s):
        call()
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph, stream=s):
        call()
    for _ in range(2):
        y.fill_(NAN)
        graph.replay()
        torch.cuda.synchronize()
        assert torch.equal(y, direct)
    o.close()
    closed.close()


@pytest.mark.parametrize("op", [0, 1, 2], ids=["N", "T", "C"])
def test_forwarded_complex_calls_are_counted(L, op):
    """a double-complex CSR SpMV outside the routed cases goes to the closed library, counted as forwarded, with its result"""
    from cudalibrarysamples_b200 import cusparse_api as cs
    m = 4096
    arrays, x = shim_case(m, 8, seed=2)
    assert L.b200spmv_route(1, op, 0, 2, 2, 5, 5, 5, 5, m, m, arrays["col"].numel()) == 0
    api = cs.Api("b200")
    api.reset_stats()
    o = cs.SpMVOperator(api, "csr", m, m, arrays, op=op)
    y = torch.zeros(m, dtype=torch.complex128, device=DEV)
    o(x, y, 0.5 + 1j)
    torch.cuda.synchronize()
    st = api.stats()
    assert st["native"] == 0 and st["forwarded"] == 1, st
    closed = cs.SpMVOperator(cs.Api("cusparse"), "csr", m, m, arrays, op=op)
    yc = torch.zeros(m, dtype=torch.complex128, device=DEV)
    closed(x, yc, 0.5 + 1j)
    torch.cuda.synchronize()
    assert rel_err(y, yc, arrays, x, op) < 3000 * 2.0 ** -48
    o.close()
    closed.close()
