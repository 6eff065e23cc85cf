"""GPU: the shim's double-complex SpMV path (ZCSR) run for real with B200SPMV_ZCSR=on -- bufferSize, preprocess, the counted native
call for opA N / T / C, graph capture, a misaligned complex view kept from the kernel -- and the split walk's carry slots written exactly
as the walk model (oracle/spmv_csr16_ref.walk, which the complex kernel shares) says."""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import spmv_csr_z_ref as R

pytestmark = pytest.mark.gpu

DEV = "cuda"
C64 = 5
NAN = complex(float("nan"), float("nan"))


@pytest.fixture(scope="module")
def L():
    from cudalibrarysamples_b200 import lib
    return lib.shim()


@pytest.fixture
def zcsr_on(L):
    assert L.b200spmv_set_option(b"B200SPMV_ZCSR", b"on") == 0
    try:
        yield
    finally:
        assert L.b200spmv_set_option(b"B200SPMV_ZCSR", b"auto") == 0


def case(m, per, seed):
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
    y0 = torch.complex(torch.rand(m, device=DEV, generator=g, dtype=torch.float64) - 0.5,
                       torch.rand(m, device=DEV, generator=g, dtype=torch.float64) - 0.5)
    return dict(off=off, col=col, val=val), x, y0


def magnitude(arrays, x, op):
    """sum |a| |x| per entry of y (rows for N, columns for T / C)"""
    off, col, val = arrays["off"], arrays["col"], arrays["val"]
    m = off.numel() - 1
    row = torch.repeat_interleave(torch.arange(m, device=DEV), (off[1:] - off[:-1]).long())
    src, dst = (col.long(), row) if op == 0 else (row, col.long())
    return torch.zeros(m, dtype=torch.float64, device=DEV).index_add_(0, dst, val.abs() * x.abs()[src])


def direct(L, op, m, arrays, x, y, alpha, beta, ws=None, wsb=0):
    from cudalibrarysamples_b200.cusparse_api import CDoubleComplex
    a, b = CDoubleComplex(alpha), CDoubleComplex(beta)
    rc = L.b200spmv_csr_z(torch.cuda.current_stream().cuda_stream, op, m, m, arrays["col"].numel(), arrays["off"].data_ptr(),
                          arrays["col"].data_ptr(), arrays["val"].data_ptr(), 0, C.addressof(a), C.addressof(b), 0, x.data_ptr(),
                          y.data_ptr(), ws, wsb)
    torch.cuda.synchronize()
    assert rc == 0, rc


@pytest.mark.parametrize("op", [0, 1, 2], ids=["N", "T", "C"])
def test_shim_serves_the_class_natively_when_switched_on(L, zcsr_on, op):
    """route 4 over the same descriptors; bufferSize >= the closed library's and ours; preprocess succeeds without an analysis; the
    call is counted native and names the kernel; y equals b200spmv_csr_z's (bit for bit for N, within fp64 tolerance for the
    atomics of T / C) and the closed library's within tolerance"""
    from cudalibrarysamples_b200 import cusparse_api as cs
    m = 1 << 15
    arrays, x, y0 = case(m, 9, seed=op + 1)
    nnz = arrays["col"].numel()
    alpha, beta = 0.75 + 0.5j, 0.5 - 0.25j
    assert L.b200spmv_route(1, op, 0, 2, 2, C64, C64, C64, C64, m, m, nnz) == 4
    closed = cs.SpMVOperator(cs.Api("cusparse"), "csr", m, m, arrays, op=op)
    yc = y0.clone()
    closed(x, yc, alpha, beta)
    api = cs.Api("b200")
    api.reset_stats()
    o = cs.SpMVOperator(api, "csr", m, m, arrays, op=op)            # bufferSize, then preprocess
    assert o.buffer_bytes >= closed.buffer_bytes
    if op == 0:
        assert o.buffer_bytes >= L.b200spmv_csr_z_workspace_bytes(m, nnz)
    assert L.b200spmv_csr16_route(o.mat, o.vecX, o.vecY, op, C64, 0) == 4
    y = y0.clone()
    o(x, y, alpha, beta)
    torch.cuda.synchronize()
    st = api.stats()
    assert st == dict(native=1, forwarded=0, analyze=0), st
    assert api.last_csr_kernel() == ("b200::spmv_csrz_chunk_kernel" if op == 0 else "b200::spmv_csrz_transpose_kernel")
    want = y0.clone()
    wsb = L.b200spmv_csr_z_workspace_bytes(m, nnz) if op == 0 else 0
    direct(L, op, m, arrays, x, want, alpha, beta, o.buffer.data_ptr() if op == 0 else None, wsb)
    bound = abs(alpha) * magnitude(arrays, x, op) + abs(beta) * y0.abs() + 1e-300
    tol = 3100 * 4 * 2.0 ** -52
    if op == 0:
        assert torch.equal(y, want)
    else:
        assert (((y - want).abs() / bound).max().item()) <= tol
    assert (((y - yc).abs() / bound).max().item()) <= 2 * tol
    o.close()
    closed.close()


def test_shim_native_call_replays_in_a_graph(L, zcsr_on):
    from cudalibrarysamples_b200 import cusparse_api as cs
    m = 1 << 14
    arrays, x, _ = case(m, 12, seed=7)
    api = cs.Api("b200")
    o = cs.SpMVOperator(api, "csr", m, m, arrays)
    y = torch.full((m,), NAN, dtype=torch.complex128, device=DEV)
    s = torch.cuda.Stream()
    api.cusparseSetStream(o.handle, s.cuda_stream)
    call = o.prebuilt(x, y, 1 - 1j)
    with torch.cuda.stream(s):
        call()
    torch.cuda.synchronize()
    first = y.clone()
    assert torch.isfinite(first.real).all() and torch.isfinite(first.imag).all()
    graph = torch.cuda.CUDAGraph()
    api.reset_stats()
    with torch.cuda.graph(graph, stream=s):
        call()
    assert api.stats()["forwarded"] == 0
    for _ in range(2):
        y.fill_(NAN)
        graph.replay()
        torch.cuda.synchronize()
        assert torch.equal(y, first)
    o.close()


def test_a_misaligned_complex_view_never_reaches_the_kernel(L, zcsr_on):
    """a y of doubles 8 bytes off a 16-byte boundary: the closed library refuses such a CUDA_C_64F vector at creation.  If
    cusparseDnVecSetValues lets one through, cusparseSpMV hands the call to the closed library (counted forwarded), never to
    b200spmv_csr_z"""
    from cudalibrarysamples_b200 import cusparse_api as cs
    m = 4096
    arrays, x, _ = case(m, 8, seed=9)
    api = cs.Api("b200")
    o = cs.SpMVOperator(api, "csr", m, m, arrays)
    raw = torch.zeros(2 * m + 2, dtype=torch.float64, device=DEV)
    view = raw[1:1 + 2 * m]                                          # 8 bytes off
    assert view.data_ptr() % 16 == 8
    h = C.c_void_p()
    assert api.lib.cusparseCreateDnVec(C.byref(h), C.c_int64(m), C.c_void_p(view.data_ptr()), C64) != 0
    y = torch.zeros(m, dtype=torch.complex128, device=DEV)
    assert api.lib.cusparseDnVecSetValues(o.vecX, C.c_void_p(x.data_ptr())) == 0
    if api.lib.cusparseDnVecSetValues(o.vecY, C.c_void_p(view.data_ptr())) != 0:
        o.close()
        return                                                       # refused here too: no misaligned view exists
    api.reset_stats()
    pa, pb = cs.CDoubleComplex(1 + 1j), cs.CDoubleComplex(0)
    api.lib.cusparseSpMV(o.handle, 0, C.byref(pa), o.mat, o.vecX, C.byref(pb), o.vecY, C64, 0, C.c_void_p(o.buffer.data_ptr()))
    torch.cuda.synchronize()
    assert api.stats()["native"] == 0 and api.stats()["forwarded"] == 1, api.stats()
    assert api.lib.cusparseDnVecSetValues(o.vecY, C.c_void_p(y.data_ptr())) == 0
    o.close()


@pytest.mark.parametrize("name", ["edges", "long", "one-row", "many-short", "trailing-empty"])
def test_split_walk_writes_the_carry_slots_of_the_walk_model(L, name):
    """the workspace starts as a sentinel; after the split walk exactly the slots the walk model writes differ from it"""
    E = R.params(L)["chunk"]
    lengths = {"edges": [0, 1, E - 1, E, E + 1, 0, 2 * E - 1, 2 * E + 1, 3, E, 0, 2 * E - 1, 2 * E + 1, 1],
               "long": [5, 40 * E + 17, 0, 2, E + 1], "one-row": [3 * E + 7], "many-short": [1, 2, 3, 0, 30, 31, 32, 33] * 40,
               "trailing-empty": [E, E, 0, 0, 0]}[name]
    k = max(lengths) + 8
    off, col = R.pattern(lengths, k, seed=3)
    val, x, _ = R.values(len(lengths), k, len(col), seed=4)
    rows, nnz = len(lengths), len(col)
    arrays = dict(off=torch.tensor(off, dtype=torch.int32, device=DEV), col=torch.tensor(col, dtype=torch.int32, device=DEV),
                  val=torch.tensor(val, dtype=torch.complex128, device=DEV))
    xd = torch.tensor(x, dtype=torch.complex128, device=DEV)
    wsb = L.b200spmv_csr_z_workspace_bytes(rows, nnz)
    ws = torch.full((wsb,), 0x7F, dtype=torch.uint8, device=DEV)
    y = torch.full((rows,), NAN, dtype=torch.complex128, device=DEV)
    from cudalibrarysamples_b200.cusparse_api import CDoubleComplex
    a, b = CDoubleComplex(1), CDoubleComplex(0)
    assert L.b200spmv_csr_z(torch.cuda.current_stream().cuda_stream, 0, rows, k, nnz, arrays["off"].data_ptr(), arrays["col"].data_ptr(),
                            arrays["val"].data_ptr(), 0, C.addressof(a), C.addressof(b), 0, xd.data_ptr(), y.data_ptr(), ws.data_ptr(),
                            wsb) == 0
    torch.cuda.synchronize()
    slots = ws.cpu().numpy().reshape(-1, 16)
    written = set(np.flatnonzero((slots != 0x7F).any(axis=1)).tolist())
    writes, reads, _ = R.walk(np.asarray(off), E, split=True)
    model = {w[1] for w in writes if w[0] == "carry"}
    assert written == model, (sorted(written - model)[:10], sorted(model - written)[:10])
    assert sorted(r[1] for r in reads) == sorted(model)                 # each written slot is read once by the fix-up
    assert np.array_equal(y.cpu().numpy(), R.reference_int(off, col, val, x, None, 1, 0))
