"""GPU: b200spmm_csr_t -- the transposed plan read back against scipy's tocsc(), its determinism across builds and graph replays, bit
equality with the opA = N entry points on the explicit transpose, exact integer results, and cusparseSpMM with opA = T / C through
the shim against the closed library."""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import exact as X
from oracle import oracle as O
from oracle import spmm_csr16_ref as HR
from oracle import spmm_csr_t_ref as T

pytestmark = pytest.mark.gpu

F32, F64, F16, BF16 = 0, 1, 2, 14
TD = {F32: torch.float32, F64: torch.float64, F16: torch.float16, BF16: torch.bfloat16}
ROW, COL = 2, 1
NT, TR, CT = 0, 1, 2


@pytest.fixture(scope="module")
def L():
    if not torch.cuda.is_available():
        pytest.skip("no GPU")
    from cudalibrarysamples_b200 import lib
    return lib.shim()


@pytest.fixture(scope="module")
def N(L):
    """b200spmm_csr_ws / b200spmm_csr_workspace_bytes with 64-bit arguments, on a handle of its own"""
    from cudalibrarysamples_b200 import build, lib
    return lib.load(build.LIB_PATH)


def dev(a, dtype=None):
    return torch.tensor(np.asarray(a), device="cuda", dtype=dtype)


def bits(t):
    return t.reshape(-1).view({2: torch.int16, 4: torch.int32, 8: torch.int64}[t.element_size()])


def stream():
    return torch.cuda.current_stream().cuda_stream


def skewed(rows, cols, seed, hub_len=1500):
    """a pattern whose columns 0 and 7 are stored by hub_len rows each (A^T rows longer than a csr16 piece), the rest random"""
    rng = np.random.default_rng(seed)
    per = [set(rng.choice(cols, rng.integers(0, 6), replace=False).tolist()) for _ in range(rows)]
    for r in rng.choice(rows, hub_len, replace=False):
        per[r] |= {0, 7}
    off = np.concatenate([[0], np.cumsum([len(s) for s in per])])
    col = np.concatenate([sorted(s) for s in per]).astype(np.int64)
    return off, col


def patterns():
    off, col, _ = O.rmat_csr(3000, avg_nnz=8, seed=3, val_seed=4)
    yield "rmat", off, col, 3000, 3000
    off, col = skewed(2000, 300, 5)
    yield "skew", off, col, 2000, 300
    off, col, _ = O.rmat_csr(2000, cols=70000, avg_nnz=4, seed=6, val_seed=7)
    yield "wide", off, col, 2000, 70000
    off, col, _ = O.gen_stencil5(30)
    yield "stencil", off, col, len(off) - 1, len(off) - 1
    yield "empty", np.zeros(6, np.int64), np.zeros(0, np.int64), 5, 4


def layout(L, dt, rows, cols, n, nnz, sbk, sbj):
    offs = (C.c_size_t * 6)()
    total = L.b200spmm_csr_t_layout(dt, rows, cols, n, nnz, sbk, sbj, offs)
    return total, list(offs)


def read_plan(ws, offs, cols, nnz):
    i = lambda o, k: ws[o:o + 4 * k].view(torch.int32).cpu().numpy().astype(np.int64)      # noqa: E731
    return i(offs[0], cols + 1), i(offs[1], nnz), i(offs[2], nnz)


@pytest.mark.parametrize("base", [0, 1])
def test_plan_equals_tocsc_and_is_deterministic(L, base):
    for name, off, col, rows, cols in patterns():
        nnz = len(col)
        total, offs = layout(L, F32, rows, cols, 8, nnz, 8, 1)
        o, c = dev(np.asarray(off) + base, torch.int32), dev(np.asarray(col) + base, torch.int32)
        want = T.plan_scipy(off, col, rows, cols)
        plans = []
        for fill in (0x00, 0x7F):
            ws = torch.full((total,), fill, dtype=torch.uint8, device="cuda")
            assert L.b200spmm_csr_t_plan(stream(), rows, cols, nnz, o.data_ptr(), c.data_ptr(), base, ws.data_ptr(), offs[4]) == 0
            torch.cuda.synchronize()
            got = read_plan(ws, offs, cols, nnz)
            for g, w, what in zip(got, want, ("tOff", "tRow", "perm")):
                assert np.array_equal(g, w), (name, what)
            plans.append([ws[offs[0]:offs[0] + 4 * (cols + 1)].clone(), ws[offs[1]:offs[1] + 4 * nnz].clone(),
                          ws[offs[2]:offs[2] + 4 * nnz].clone()])
        assert all(torch.equal(x, y) for x, y in zip(*plans)), name       # two builds over different stale bytes: identical plans


def test_plan_in_a_graph_replays_identically(L):
    off, col, _ = O.rmat_csr(5000, avg_nnz=8, seed=11, val_seed=12)
    rows = cols = 5000
    nnz = len(col)
    total, offs = layout(L, F32, rows, cols, 8, nnz, 8, 1)
    o, c = dev(off, torch.int32), dev(col, torch.int32)
    ws = torch.zeros(total, dtype=torch.uint8, device="cuda")
    s = torch.cuda.Stream()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s):
        with torch.cuda.graph(g, stream=s):
            assert L.b200spmm_csr_t_plan(s.cuda_stream, rows, cols, nnz, o.data_ptr(), c.data_ptr(), 0, ws.data_ptr(), offs[4]) == 0
    want = T.plan_scipy(off, col, rows, cols)
    for _ in range(2):
        ws.fill_(0x55)
        g.replay()
        torch.cuda.synchronize()
        for gg, w in zip(read_plan(ws, offs, cols, nnz), want):
            assert np.array_equal(gg, w)


def values(dt, nnz, rows, cols, n, seed):
    rng = np.random.default_rng(seed)
    val = rng.standard_normal(nnz)
    B = rng.standard_normal((rows, n))
    C0 = rng.standard_normal((cols, n))
    return val, B, C0


def call_t(L, dt, ct, rows, cols, n, o, c, v, base, alpha, beta, on_dev, Bs, sbk, sbj, Cb, ldc, crow, plan_valid, ws):
    return L.b200spmm_csr_t(stream(), dt, ct, rows, cols, n, c.numel(), o.data_ptr(), c.data_ptr(), v.data_ptr(), base, alpha, beta,
                            on_dev, Bs.data_ptr(), sbk, sbj, Cb.data_ptr(), ldc, crow, plan_valid, ws.data_ptr(), ws.numel())


def scalars(ct, alpha, beta, on_dev):
    if on_dev:
        td = torch.float64 if ct == F64 else torch.float32
        a, b = torch.tensor([alpha], dtype=td, device="cuda"), torch.tensor([beta], dtype=td, device="cuda")
        return (a, b), a.data_ptr(), b.data_ptr()
    h = (C.c_double(alpha), C.c_double(beta)) if ct == F64 else (C.c_float(alpha), C.c_float(beta))
    return h, C.addressof(h[0]), C.addressof(h[1])


CASES = [(dt, ct, ob, oc, opb) for dt, ct in ((F32, F32), (F64, F64)) for ob in (ROW, COL) for oc in (ROW, COL) for opb in (NT,)] + \
        [(dt, ct, ob, oc, opb) for dt, ct in ((F16, F16), (F16, F32), (BF16, BF16), (BF16, F32)) for ob in (ROW, COL) for oc in (ROW, COL)
         for opb in (NT, TR)]


@pytest.mark.parametrize("dt,ct,ob,oc,opb", CASES)
def test_bit_equal_to_the_n_kernels_on_the_explicit_transpose(L, N, dt, ct, ob, oc, opb):
    n = 40
    for (name, off, col, rows, cols), base, on_dev, beta in zip(list(patterns())[:3], (0, 1, 0), (0, 1, 0), (0.5, 0.0, -1.0)):
        nnz = len(col)
        val, B, C0 = values(dt, nnz, rows, cols, n, 7)
        vt, ctd = TD[dt], TD[ct]
        o, c, v = dev(np.asarray(off) + base, torch.int32), dev(np.asarray(col) + base, torch.int32), dev(val, vt)
        t_off, t_row, perm = T.plan(off, col, cols)
        to, tr = dev(t_off, torch.int32), dev(t_row, torch.int32)
        tv = v[dev(perm, torch.int64)]                        # the values of A^T in CSC order
        Bt = dev(B, vt)                                       # op(B), rows x n
        if opb == NT:
            Bs = Bt.contiguous() if ob == ROW else Bt.t().contiguous()
            sbk, sbj = (n, 1) if ob == ROW else (1, rows)
        else:                                                 # B holds the n x rows matrix whose transpose is op(B)
            Bs = Bt.t().contiguous() if ob == ROW else Bt.contiguous()
            sbk, sbj = (1, rows) if ob == ROW else (n, 1)
        crow = 1 if oc == ROW else 0
        ldc = n if crow else cols
        C0s = dev(C0, ctd)
        C0s = C0s.contiguous() if crow else C0s.t().contiguous()
        if beta == 0.0:
            C0s = torch.full_like(C0s, float("nan"))          # beta = 0 must not read C
        keep, pa, pb = scalars(ct, 1.5, beta, on_dev)
        ours = C0s.clone()
        total = L.b200spmm_csr_t_workspace_bytes(dt, rows, cols, n, nnz, sbk, sbj)
        ws = torch.full((total,), 0x3C, dtype=torch.uint8, device="cuda")
        assert call_t(L, dt, ct, rows, cols, n, o, c, v, base, pa, pb, on_dev, Bs, sbk, sbj, ours, ldc, crow, 0, ws) == 0
        ref = C0s.clone()
        if dt in (F32, F64):
            nws = N.b200spmm_csr_workspace_bytes(dt, rows, n, 1 if sbj == 1 else 0)
            w2 = torch.empty(max(nws, 16), dtype=torch.uint8, device="cuda")
            rc = N.b200spmm_csr_ws(stream(), dt, cols, rows, n, nnz, to.data_ptr(), tr.data_ptr(), tv.data_ptr(), 0, pa, pb, on_dev,
                                   Bs.data_ptr(), sbk if sbj == 1 else sbj, 1 if sbj == 1 else 0, ref.data_ptr(), ldc, crow, w2.data_ptr())
        else:
            nws = L.b200spmm_csr16_workspace_bytes(rows, n, nnz, sbk, sbj)
            w2 = torch.empty(max(nws, 16), dtype=torch.uint8, device="cuda")
            rc = L.b200spmm_csr16(stream(), dt, ct, cols, rows, n, nnz, to.data_ptr(), tr.data_ptr(), tv.data_ptr(), 0, pa, pb, on_dev,
                                  Bs.data_ptr(), sbk, sbj, ref.data_ptr(), ldc, crow, w2.data_ptr(), nws)
        assert rc == 0
        torch.cuda.synchronize()
        assert torch.equal(bits(ours), bits(ref)), name
        assert not torch.isnan(ours).any(), name
        # a second call on the plan the first one built: new values gathered, same bits as a call that rebuilds
        v2 = -v
        again, rebuilt = C0s.clone(), C0s.clone()
        assert call_t(L, dt, ct, rows, cols, n, o, c, v2, base, pa, pb, on_dev, Bs, sbk, sbj, again, ldc, crow, 1, ws) == 0
        assert call_t(L, dt, ct, rows, cols, n, o, c, v2, base, pa, pb, on_dev, Bs, sbk, sbj, rebuilt, ldc, crow, 0, ws) == 0
        torch.cuda.synchronize()
        assert torch.equal(bits(again), bits(rebuilt)), name
        del keep


@pytest.mark.parametrize("dt", [F32, F64])
def test_integer_data_is_exact(L, dt):
    off, col = skewed(1500, 200, 9)
    rows, cols, n = 1500, 200, 24
    nnz = len(col)
    rng = np.random.default_rng(1)
    a = X.nonzero_ints(rng, nnz, 1, 3)
    B = X.nonzero_ints(rng, rows * n, 1, 4).reshape(rows, n)
    C0 = rng.integers(-4, 5, (cols, n)).astype(np.int64)
    p = 24 if dt == F32 else 53
    t_off, t_row, t_val = T.transpose(off, col, a, rows, cols)
    X.check_spmm_exact(t_off, t_row, t_val, B, C0, p)
    for alpha, beta in X.SCALARS:
        want = X.spmm_reference(t_off, t_row, t_val, B, C0, alpha, beta)
        vt = TD[dt]
        o, c, v = dev(off, torch.int32), dev(col, torch.int32), dev(a, vt)
        Bs = dev(B, vt).t().contiguous()                      # column-major, the samples' layout
        Cs = dev(C0, vt).t().contiguous()
        keep, pa, pb = scalars(dt, alpha, beta, 0)
        ws = torch.empty(L.b200spmm_csr_t_workspace_bytes(dt, rows, cols, n, nnz, 1, rows), dtype=torch.uint8, device="cuda")
        assert call_t(L, dt, dt, rows, cols, n, o, c, v, 0, pa, pb, 0, Bs, 1, rows, Cs, cols, 0, 0, ws) == 0
        torch.cuda.synchronize()
        assert np.array_equal(Cs.t().cpu().numpy(), want), (alpha, beta)


@pytest.mark.parametrize("dt,ct", [(F16, F32), (BF16, BF16)])
def test_integer_data_is_exact_16bit(L, dt, ct):
    off, col = skewed(1200, 64, 4, hub_len=1100)             # columns 0 and 7: A^T rows of 1100 entries, split into pieces
    rows, cols, n = 1200, 64, 16
    nnz = len(col)
    val, Bv, _ = HR.values(cols, rows, n, nnz, seed=3)
    t_off, t_row, t_val = T.transpose(off, col, val, rows, cols)
    want = HR.reference_int(t_off, t_row, t_val, Bv, None, 1.0, 0.0, "f32" if ct == F32 else "bf16")
    o, c, v = dev(off, torch.int32), dev(col, torch.int32), dev(val, TD[dt])
    Bs = dev(Bv, TD[dt]).contiguous()
    Cs = torch.full((cols, n), float("nan"), dtype=TD[ct], device="cuda")
    keep, pa, pb = scalars(F32, 1.0, 0.0, 0)
    ws = torch.empty(L.b200spmm_csr_t_workspace_bytes(dt, rows, cols, n, nnz, n, 1), dtype=torch.uint8, device="cuda")
    assert call_t(L, dt, ct, rows, cols, n, o, c, v, 0, pa, pb, 0, Bs, n, 1, Cs, n, 1, 0, ws) == 0
    torch.cuda.synchronize()
    assert np.array_equal(Cs.double().cpu().numpy(), want)


# ---------------------------------------------------------------- through the shim
@pytest.fixture(scope="module")
def api(L):
    from cudalibrarysamples_b200 import cusparse_api as cs
    return cs.Api("b200")


def close_to(got, want, scale, tol):
    """|got - want| <= tol * max |want| (the closed library's transpose adds in no fixed order)"""
    return float((got.double() - want.double()).abs().max()) <= tol * max(float(want.double().abs().max()), scale)


@pytest.mark.parametrize("dt", [F32, F64, F16])
@pytest.mark.parametrize("preprocess", [True, False])
def test_shim_forwards_unmeasured_classes_and_counts_them(L, api, dt, preprocess):
    """a 4000-row R-MAT is outside every measured class: the call goes to the closed library, counted; opA = C is refused as the
    closed library refuses it for real types"""
    from cudalibrarysamples_b200 import cusparse_api as cs
    off, col, _ = O.rmat_csr(4000, avg_nnz=8, seed=21, val_seed=22)
    rows = cols = 4000
    n = 32
    val, B, C0 = values(dt, len(col), rows, cols, n, 3)
    vt = TD[dt]
    arrays = dict(off=dev(off, torch.int32), col=dev(col, torch.int32), val=dev(val, vt))
    Bc = dev(B, vt).t().contiguous().view(-1)
    Cc = dev(C0, vt).t().contiguous().view(-1)
    api.reset_stats()
    got = cs.spmm(api, rows, cols, arrays, Bc, Cc, 1.0, 0.5, op_a=TR, n=n, preprocess=preprocess)
    st = api.stats()
    assert st["forwarded"] == 1 and st["native"] == 0, st
    closed = cs.spmm(cs.Api("cusparse"), rows, cols, arrays, Bc, Cc, 1.0, 0.5, op_a=TR, n=n)
    assert close_to(got, closed, 1.0, {F32: 1e-5, F64: 1e-13, F16: 1e-2}[dt])
    with pytest.raises(cs.CuSparseError):
        cs.spmm(api, rows, cols, arrays, Bc, Cc, 1.0, 0.5, op_a=CT, n=n, preprocess=preprocess)


def uniform16(rows, seed):
    """rows x rows, 16 entries per row at random columns: inside the measured classes"""
    g = torch.Generator(device="cuda").manual_seed(seed)
    col = torch.randint(0, rows, (rows * 16,), device="cuda", generator=g, dtype=torch.int32)
    col = col.view(rows, 16).sort(dim=1).values.reshape(-1).contiguous()
    off = torch.arange(0, rows * 16 + 1, 16, device="cuda", dtype=torch.int32)
    return off, col, g


ROUTED = [(F32, COL, 64, True), (F32, COL, 64, False), (F64, COL, 128, True), (F16, ROW, 32, True), (BF16, COL, 32, False)]


@pytest.mark.parametrize("dt,order,n,preprocess", ROUTED)
def test_shim_routes_measured_classes_natively(L, api, dt, order, n, preprocess):
    from cudalibrarysamples_b200 import cusparse_api as cs
    rows = 1 << 20
    off, col, g = uniform16(rows, 8)
    vt = TD[dt]
    val = (torch.rand(col.numel(), device="cuda", generator=g) * 2 - 1).to(vt)
    B = (torch.rand(rows * n, device="cuda", generator=g) * 2 - 1).to(vt)
    C0 = (torch.rand(rows * n, device="cuda", generator=g) * 2 - 1).to(vt)
    arrays = dict(off=off, col=col, val=val)
    api.reset_stats()
    got = cs.spmm(api, rows, rows, arrays, B, C0, 1.0, 0.5, op_a=TR, n=n, order_b=order, order_c=order, preprocess=preprocess)
    st = api.stats()
    assert st["forwarded"] == 0 and st["native"] == 1, st
    closed = cs.spmm(cs.Api("cusparse"), rows, rows, arrays, B, C0, 1.0, 0.5, op_a=TR, n=n, order_b=order, order_c=order)
    assert close_to(got, closed, 1.0, {F32: 1e-5, F64: 1e-13, F16: 1e-2, BF16: 5e-2}[dt])
    # bit for bit what b200spmm_csr_t gives on the same operands (deterministic: no atomics)
    sbk, sbj = (n, 1) if order == ROW else (1, rows)
    ws = torch.empty(L.b200spmm_csr_t_workspace_bytes(dt, rows, rows, n, col.numel(), sbk, sbj), dtype=torch.uint8, device="cuda")
    keep, pa, pb = scalars(F64 if dt == F64 else F32, 1.0, 0.5, 0)
    direct = C0.clone()
    assert call_t(L, dt, dt, rows, rows, n, off, col, val, 0, pa, pb, 0, B, sbk, sbj, direct, n if order == ROW else rows,
                  1 if order == ROW else 0, 0, ws) == 0
    torch.cuda.synchronize()
    assert torch.equal(bits(got), bits(direct))


def test_shim_plan_follows_set_values_and_set_pointers(L, api):
    """one handle, one buffer, preprocess once: new values on the same plan, then new pointers (a new pattern) with a rebuilt plan"""
    from cudalibrarysamples_b200 import cusparse_api as cs
    rows, n = 1 << 20, 64
    off, col, g = uniform16(rows, 9)
    val = torch.rand(col.numel(), device="cuda", generator=g) * 2 - 1
    B = torch.rand(rows * n, device="cuda", generator=g) * 2 - 1
    Cb = torch.zeros(rows * n, device="cuda")
    h = api.cusparseCreate()
    mat = api.cusparseCreateCsr(rows, rows, col.numel(), off, col, val, 0)
    mB = api.cusparseCreateDnMat(rows, n, rows, B, COL)
    mC = api.cusparseCreateDnMat(rows, n, rows, Cb, COL)
    ref = cs.Api("cusparse")
    try:
        size = api.cusparseSpMM_bufferSize(h, TR, NT, 1.0, mat, mB, 0.0, mC, 0, 0)
        buf = torch.empty(size, dtype=torch.uint8, device="cuda")
        api.cusparseSpMM_preprocess(h, TR, NT, 1.0, mat, mB, 0.0, mC, 0, 0, buf)
        assert L.b200spmv_plan_trusted(mat, C.c_void_p(buf.data_ptr()), 1) == 1
        api.reset_stats()
        val2 = -2 * val
        api.cusparseSpMatSetValues(mat, val2)
        api.cusparseSpMM(h, TR, NT, 1.0, mat, mB, 0.0, mC, 0, 0, buf)
        torch.cuda.synchronize()
        want = cs.spmm(ref, rows, rows, dict(off=off, col=col, val=val2), B, torch.zeros_like(Cb), 1.0, 0.0, op_a=TR, n=n)
        assert close_to(Cb, want, 1.0, 1e-5)
        off2, col2, _ = uniform16(rows, 10)
        api.cusparseCsrSetPointers(mat, off2, col2, val)
        assert L.b200spmv_plan_trusted(mat, C.c_void_p(buf.data_ptr()), 1) == 0
        api.cusparseSpMM(h, TR, NT, 1.0, mat, mB, 0.0, mC, 0, 0, buf)
        torch.cuda.synchronize()
        want = cs.spmm(ref, rows, rows, dict(off=off2, col=col2, val=val), B, torch.zeros_like(Cb), 1.0, 0.0, op_a=TR, n=n)
        assert close_to(Cb, want, 1.0, 1e-5)
        st = api.stats()
        assert st["forwarded"] == 0 and st["native"] == 2, st
    finally:
        api.cusparseDestroySpMat(mat)
        api.cusparseDestroyDnMat(mB)
        api.cusparseDestroyDnMat(mC)
        api.cusparseDestroy(h)


def test_spmv_plan_is_not_trusted_as_a_transposed_plan(L, api):
    """preprocess a CSR SpMV on a buffer; the same matrix's transposed SpMM must not find its plan there"""
    from cudalibrarysamples_b200 import cusparse_api as cs
    off, col, val = O.rmat_csr(3000, avg_nnz=16, seed=31, val_seed=32)
    arrays = dict(off=dev(off, torch.int32), col=dev(col, torch.int32), val=dev(val, torch.float64))
    op = cs.SpMVOperator(api, "csr", 3000, 3000, arrays, preprocess=True)
    try:
        mat, buf = op.mat, op.buffer
        ptr = C.c_void_p(buf.data_ptr())
        assert L.b200spmv_plan_trusted(mat, ptr, 0) == 1
        assert L.b200spmv_plan_trusted(mat, ptr, 1) == 0
    finally:
        op.close()


def test_buffer_preprocessed_for_spmv_is_not_trusted_by_a_routed_spmm(L, api):
    """one matrix, one buffer: SpMV preprocess then SpMM, which must rebuild its plan (and still be right)"""
    from cudalibrarysamples_b200 import cusparse_api as cs
    rows, n = 1 << 20, 64
    off, col, g = uniform16(rows, 11)
    val = torch.rand(col.numel(), device="cuda", generator=g) * 2 - 1
    B = torch.rand(rows * n, device="cuda", generator=g) * 2 - 1
    Cb = torch.zeros(rows * n, device="cuda")
    x, y = torch.ones(rows, device="cuda"), torch.zeros(rows, device="cuda")
    h = api.cusparseCreate()
    mat = api.cusparseCreateCsr(rows, rows, col.numel(), off, col, val, 0)
    mB = api.cusparseCreateDnMat(rows, n, rows, B, COL)
    mC = api.cusparseCreateDnMat(rows, n, rows, Cb, COL)
    vx, vy = api.cusparseCreateDnVec(rows, x), api.cusparseCreateDnVec(rows, y)
    try:
        size = max(api.cusparseSpMM_bufferSize(h, TR, NT, 1.0, mat, mB, 0.0, mC, 0, 0),
                   api.cusparseSpMV_bufferSize(h, NT, 1.0, mat, vx, 0.0, vy, 0, 0))
        buf = torch.empty(size, dtype=torch.uint8, device="cuda")
        api.cusparseSpMM_preprocess(h, TR, NT, 1.0, mat, mB, 0.0, mC, 0, 0, buf)
        api.cusparseSpMV_preprocess(h, NT, 1.0, mat, vx, 0.0, vy, 0, 0, buf)       # overwrites the buffer with the SpMV plan
        ptr = C.c_void_p(buf.data_ptr())
        assert L.b200spmv_plan_trusted(mat, ptr, 1) == 0 and L.b200spmv_plan_trusted(mat, ptr, 0) == 1
        api.reset_stats()
        api.cusparseSpMM(h, TR, NT, 1.0, mat, mB, 0.0, mC, 0, 0, buf)
        torch.cuda.synchronize()
        assert api.stats()["native"] == 1
        want = cs.spmm(cs.Api("cusparse"), rows, rows, dict(off=off, col=col, val=val), B, torch.zeros_like(Cb), 1.0, 0.0, op_a=TR, n=n)
        assert close_to(Cb, want, 1.0, 1e-5)
    finally:
        for d in (vx, vy):
            api.cusparseDestroyDnVec(d)
        api.cusparseDestroySpMat(mat)
        api.cusparseDestroyDnMat(mB)
        api.cusparseDestroyDnMat(mC)
        api.cusparseDestroy(h)


@pytest.mark.parametrize("dt,order,n", [(F16, COL, 64), (BF16, ROW, 128)])
def test_shim_forwards_16bit_opb_t_at_a_routed_size(L, api, dt, order, n):
    """opB = T was not measured: at a size where opB = N is native, the call goes to the closed library and is counted"""
    from cudalibrarysamples_b200 import cusparse_api as cs
    rows = 1 << 20
    off, col, g = uniform16(rows, 12)
    vt = TD[dt]
    val = (torch.rand(col.numel(), device="cuda", generator=g) * 2 - 1).to(vt)
    B = (torch.rand(rows * n, device="cuda", generator=g) * 2 - 1).to(vt)           # holds the n x rows matrix whose transpose is op(B)
    C0 = (torch.rand(rows * n, device="cuda", generator=g) * 2 - 1).to(vt)
    arrays = dict(off=off, col=col, val=val)
    for preprocess in (True, False):
        api.reset_stats()
        got = cs.spmm(api, rows, rows, arrays, B, C0, 1.0, 0.5, op_a=TR, op_b=TR, n=n, order_b=order, order_c=order,
                      preprocess=preprocess)
        st = api.stats()
        assert st["forwarded"] == 1 and st["native"] == 0, st
        closed = cs.spmm(cs.Api("cusparse"), rows, rows, arrays, B, C0, 1.0, 0.5, op_a=TR, op_b=TR, n=n, order_b=order, order_c=order)
        assert close_to(got, closed, 1.0, {F16: 1e-2, BF16: 5e-2}[dt])


def test_other_writers_of_the_buffer_drop_the_transposed_plan(L, api):
    """preprocess A^T * B, then run A * B (native, its row-major copy of B lands in the buffer) on the same buffer: the transposed plan
    is no longer trusted, and the next A^T * B rebuilds it and is right"""
    from cudalibrarysamples_b200 import cusparse_api as cs
    rows, n = 1 << 20, 64
    off, col, g = uniform16(rows, 13)
    val = torch.rand(col.numel(), device="cuda", generator=g) * 2 - 1
    B = torch.rand(rows * n, device="cuda", generator=g) * 2 - 1
    Cb = torch.zeros(rows * n, device="cuda")
    h = api.cusparseCreate()
    mat = api.cusparseCreateCsr(rows, rows, col.numel(), off, col, val, 0)
    mB = api.cusparseCreateDnMat(rows, n, rows, B, COL)
    mC = api.cusparseCreateDnMat(rows, n, rows, Cb, COL)
    try:
        size = max(api.cusparseSpMM_bufferSize(h, TR, NT, 1.0, mat, mB, 0.0, mC, 0, 0),
                   api.cusparseSpMM_bufferSize(h, NT, NT, 1.0, mat, mB, 0.0, mC, 0, 0))
        buf = torch.empty(size, dtype=torch.uint8, device="cuda")
        ptr = C.c_void_p(buf.data_ptr())
        api.cusparseSpMM_preprocess(h, TR, NT, 1.0, mat, mB, 0.0, mC, 0, 0, buf)
        assert L.b200spmv_plan_trusted(mat, ptr, 1) == 1
        api.reset_stats()
        api.cusparseSpMM(h, NT, NT, 1.0, mat, mB, 0.0, mC, 0, 0, buf)                 # the forward product, same buffer
        assert api.stats()["native"] == 1
        assert L.b200spmv_plan_trusted(mat, ptr, 1) == 0
        api.cusparseSpMM(h, TR, NT, 1.0, mat, mB, 0.0, mC, 0, 0, buf)
        torch.cuda.synchronize()
        want = cs.spmm(cs.Api("cusparse"), rows, rows, dict(off=off, col=col, val=val), B, torch.zeros_like(Cb), 1.0, 0.0, op_a=TR, n=n)
        assert close_to(Cb, want, 1.0, 1e-5)
        assert api.stats()["native"] == 2 and api.stats()["forwarded"] == 0
    finally:
        api.cusparseDestroySpMat(mat)
        api.cusparseDestroyDnMat(mB)
        api.cusparseDestroyDnMat(mC)
        api.cusparseDestroy(h)
