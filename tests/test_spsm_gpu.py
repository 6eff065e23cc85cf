"""GPU: b200spsm_csr_analysis / _solve bit-exact against the numpy restatement (oracle/spsm_ref.py) over every axis, the plan and the
level order as the restatement states them, repeat and graph-replay identity, and cusparseSpSM through the shim against the closed
library: parity, updateMatrix, C aliasing B, the forwarded classes and the statuses."""
import ctypes as C
import itertools
import os
import subprocess

import numpy as np
import pytest
import torch

from oracle import spsm_ref as M

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ROW, COL = 2, 1
DT = {np.float32: (torch.float32, 0), np.float64: (torch.float64, 1)}


@pytest.fixture(scope="module")
def L():
    from cudalibrarysamples_b200 import lib
    return lib.shim()


def stream():
    return torch.cuda.current_stream().cuda_stream


def analyse(L, rows, off, col, base, lower, unit, tr):
    nnz = int(col.size)
    ws = torch.full((L.b200spsm_csr_workspace_bytes(rows, nnz, tr),), 0x5A, dtype=torch.uint8, device="cuda")
    offd, cold = torch.tensor(off + base, device="cuda"), torch.tensor(col + base, device="cuda")
    miss, lev = C.c_int64(-1), C.c_int64(-1)
    rc = L.b200spsm_csr_analysis(stream(), rows, nnz, offd.data_ptr(), cold.data_ptr(), base, int(lower), int(unit), int(tr), ws.data_ptr(),
                                 C.addressof(miss), C.addressof(lev))
    torch.cuda.synchronize()
    assert rc == 0
    return ws, miss.value, lev.value, (offd, cold)


def dense_buffer(A, order, pad, fill=np.nan):
    """A (r x c) stored in order with leading dimension tight + pad, padding filled: (flat array, ld)."""
    r, c = A.shape
    ld = (c if order == ROW else r) + pad
    buf = np.full(ld * (r if order == ROW else c), fill, A.dtype)
    if order == ROW:
        buf.reshape(r, ld)[:, :c] = A
    else:
        buf.reshape(c, ld)[:, :r] = A.T
    return buf, ld


def read_dense(buf, r, c, order, ld):
    return buf.reshape(r, ld)[:, :c] if order == ROW else buf.reshape(c, ld)[:, :r].T


def native_solve(L, ws, rows, nnz, val, opB, unit, opb, order_b, order_c, pad, dev_alpha, alpha, diag=None):
    """b200spsm_csr_solve on the plan in ws; returns (C rows x nrhs, C buffer, padding untouched)."""
    dtype = val.dtype.type
    tdt, code = DT[dtype]
    nrhs = opB.shape[1]
    Bs = opB if opb == 0 else opB.T
    bbuf, ldb = dense_buffer(Bs, order_b, pad)
    br, bc = (ldb, 1) if order_b == ROW else (1, ldb)
    sbi, sbk = (br, bc) if opb == 0 else (bc, br)
    cbuf, ldc = dense_buffer(np.zeros((rows, nrhs), dtype), order_c, pad)
    sci, scj = (ldc, 1) if order_c == ROW else (1, ldc)
    Bd, Cd, vd = torch.tensor(bbuf, device="cuda"), torch.tensor(cbuf, device="cuda"), torch.tensor(val, device="cuda")
    dd = torch.tensor(diag, device="cuda") if diag is not None else None
    ct = C.c_float if dtype == np.float32 else C.c_double
    ah = ct(alpha)
    ad = torch.tensor([alpha], dtype=tdt, device="cuda")
    rc = L.b200spsm_csr_solve(stream(), code, rows, nnz, int(unit), vd.data_ptr(), dd.data_ptr() if dd is not None else None,
                              ad.data_ptr() if dev_alpha else C.addressof(ah), int(dev_alpha), nrhs, Bd.data_ptr(), sbi, sbk, Cd.data_ptr(),
                              sci, scj, ws.data_ptr())
    torch.cuda.synchronize()
    assert rc == 0
    assert int(ws[8:12].view(torch.int32).item()) == 0                 # the error word: no wait ran out of budget
    out = Cd.cpu().numpy()
    pad_ok = np.isnan(out).sum() == np.isnan(cbuf).sum()           # the padding kept, no NaN result
    return read_dense(out, rows, nrhs, order_c, ldc), pad_ok, order_c == ROW or (order_c == COL and rows == 1 and pad == 0)


def plan_arrays(L, ws, rows, nnz, tr):
    o = (C.c_size_t * 10)()
    L.b200spsm_csr_layout(rows, nnz, tr, o)
    w = ws.cpu().numpy()

    def arr(k, n):
        return w[o[k]:o[k] + 4 * n].view(np.int32)
    t_off = arr(2, rows + 1)
    return dict(t_off=t_off, diag_vidx=arr(3, rows), t_col=arr(4, int(t_off[-1])), t_vidx=arr(5, int(t_off[-1])), order=arr(6, rows))


# ---------------------------------------------------------------------------------------------------- native, bit-exact
@pytest.mark.parametrize("lower,unit,tr", list(itertools.product((True, False), (False, True), (False, True))))
def test_plan_and_order_match_the_restatement(L, lower, unit, tr):
    for name, rows, off, col in M.fixtures():
        for base in (0, 1):
            ws, miss, lev, _ = analyse(L, rows, off, col, base, lower, unit, tr)
            p = M.plan(rows, off + base, col + base, base, lower, unit, tr)
            _, order, nlev = M.levels(rows, p, lower, tr)
            got = plan_arrays(L, ws, rows, int(col.size), int(tr))
            for k in ("t_off", "t_col", "t_vidx", "diag_vidx"):
                assert np.array_equal(got[k], p[k]), (name, k)
            assert np.array_equal(got["order"], order) and lev == nlev and miss == p["missing"], name


@pytest.mark.parametrize("lower,unit,tr", list(itertools.product((True, False), (False, True), (False, True))))
@pytest.mark.parametrize("opb,order_b,order_c", list(itertools.product((0, 1), (ROW, COL), (ROW, COL))))
def test_solve_bit_exact_every_layout(L, lower, unit, tr, opb, order_b, order_c):
    off, col = M.SR.stencil5_pattern(6)
    rows = 36
    rng = np.random.default_rng(int(lower) + 2 * unit + 4 * tr)
    for dtype, base, dev_alpha, nrhs in itertools.product((np.float32, np.float64), (0, 1), (False, True), (1, 2, 31, 32, 33, 100)):
        ws, _, _, _ = analyse(L, rows, off, col, base, lower, unit, tr)
        val = M.values(rows, off, col, dtype, seed=nrhs)
        opB = rng.uniform(-1, 1, (rows, nrhs)).astype(dtype)
        got, pad_ok, _ = native_solve(L, ws, rows, int(col.size), val, opB, unit, opb, order_b, order_c, 3, dev_alpha, -0.75)
        want = M.solve(rows, off + base, col + base, val, opB, -0.75, base, lower, unit, tr, M.tile(nrhs, order_c == ROW))
        assert pad_ok and np.array_equal(got, want), (dtype, base, dev_alpha, nrhs)


@pytest.mark.parametrize("name", ["toy", "stencil5_9", "chain", "diagonal", "long_rows"])
@pytest.mark.parametrize("order_c", [ROW, COL])
def test_solve_bit_exact_on_the_fixtures(L, name, order_c):
    """long_rows has rows of up to ~300 entries in every triangle, so at each nrhs (every tile width W and group count 32 / W)
    each group sums several entries and a different summation order would change the bits."""
    rows, off, col = [(r, o, c) for n, r, o, c in M.fixtures() if n == name][0]
    rng = np.random.default_rng(5)
    nrhs_set = (1, 2, 31, 32, 33, 100) if name == "long_rows" else (1, 33)
    for lower, unit, tr, dtype, nrhs in itertools.product((True, False), (False, True), (False, True), (np.float32, np.float64), nrhs_set):
        ws, _, _, _ = analyse(L, rows, off, col, 0, lower, unit, tr)
        val = M.values(rows, off, col, dtype, seed=rows)
        opB = rng.uniform(-1, 1, (rows, nrhs)).astype(dtype)
        got, pad_ok, _ = native_solve(L, ws, rows, int(col.size), val, opB, unit, 0, COL, order_c, 0, False, 1.5)
        want = M.solve(rows, off, col, val, opB, 1.5, 0, lower, unit, tr, M.tile(nrhs, order_c == ROW))
        assert pad_ok and np.array_equal(got, want), (lower, unit, tr, dtype, nrhs)


def test_toy_golden_exact(L):
    T = M.TOY_SPSM
    ws, _, lev, _ = analyse(L, 4, T["off"], T["col"], 0, True, False, False)
    got, _, _ = native_solve(L, ws, 4, 9, T["val"], T["B"].reshape(2, 4).T, False, 0, COL, COL, 0, False, 1.0)
    assert np.array_equal(got.T.ravel(), T["C_result"])


def test_updated_diagonal_is_used(L):
    off, col = M.SR.stencil5_pattern(9)
    rows = 81
    ws, _, _, _ = analyse(L, rows, off, col, 0, True, False, False)
    val = M.values(rows, off, col, np.float64, seed=2)
    diag = np.random.default_rng(1).uniform(2, 4, rows)
    opB = np.random.default_rng(2).uniform(-1, 1, (rows, 8))
    got, _, _ = native_solve(L, ws, rows, int(col.size), val, opB, False, 0, ROW, ROW, 0, False, 1.0, diag=diag)
    assert np.array_equal(got, M.solve(rows, off, col, val, opB, 1.0, w=8, diag=diag))


def test_repeats_and_graph_replays_are_bit_identical(L):
    off, col = M.SR.stencil5_pattern(40)
    rows, nnz = 1600, int(col.size)
    ws, _, _, _ = analyse(L, rows, off, col, 0, True, False, False)
    val = torch.tensor(M.values(rows, off, col, np.float64, seed=3), device="cuda")
    B = torch.rand(rows * 64, dtype=torch.float64, device="cuda")
    Cb = torch.zeros_like(B)
    one = C.c_double(1.0)

    def call():
        assert L.b200spsm_csr_solve(stream(), 1, rows, nnz, 0, val.data_ptr(), None, C.addressof(one), 0, 64, B.data_ptr(), 64, 1,
                                    Cb.data_ptr(), 64, 1, ws.data_ptr()) == 0
    call()
    torch.cuda.synchronize()
    first = Cb.clone()
    for _ in range(5):
        Cb.zero_()
        call()
    torch.cuda.synchronize()
    assert torch.equal(Cb, first)
    s = torch.cuda.Stream()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s):
        call()                                   # warm-up on the capture stream
        torch.cuda.synchronize()
        with torch.cuda.graph(g, stream=s):
            call()
    for _ in range(3):
        Cb.zero_()
        g.replay()
        torch.cuda.synchronize()
        assert torch.equal(Cb, first)
    assert int(ws[8:12].view(torch.int32).item()) == 0


# ---------------------------------------------------------------------------------------------------- through the shim
def shim_case(impl, rows, off, col, val, B, nrhs, **kw):
    from cudalibrarysamples_b200 import cusparse_api as cs
    api = cs.Api(impl)
    arr = dict(off=torch.tensor(off, device="cuda"), col=torch.tensor(col, device="cuda"), val=torch.tensor(val, device="cuda"))
    return cs.spsm(api, rows, arr, torch.tensor(B, device="cuda"), nrhs, **kw).cpu().numpy()


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("order", [ROW, COL])
@pytest.mark.parametrize("lower,unit,op_a,op_b", [(True, False, 0, 0), (False, True, 1, 1), (True, True, 1, 0), (False, False, 0, 1)])
def test_parity_with_the_closed_library(L, dtype, order, lower, unit, op_a, op_b):
    from cudalibrarysamples_b200 import cusparse_api as cs
    off, col = M.SR.stencil5_pattern(30)
    rows = 900
    val = M.values(rows, off, col, dtype, seed=4)
    for nrhs in (1, 8, 33):
        Bs = np.random.default_rng(nrhs).uniform(-1, 1, (rows, nrhs) if op_b == 0 else (nrhs, rows)).astype(dtype)
        buf, _ = dense_buffer(Bs, order, 0)
        kw = dict(fill=0 if lower else 1, diag=int(unit), op_a=op_a, op_b=op_b, order_b=order, order_c=order)
        api = cs.Api("b200")
        api.reset_spsm_stats()
        ours = shim_case("b200", rows, off, col, val, buf, nrhs, alpha=2.0, **kw)
        st = api.spsm_stats()
        ref = shim_case("cusparse", rows, off, col, val, buf, nrhs, alpha=2.0, **kw)
        tol = 1e-5 if dtype == np.float32 else 1e-12
        assert np.allclose(ours, ref, rtol=tol, atol=tol), nrhs
        # no class is routed natively (DESIGN.md 3.20): analysis and solve are forwarded and counted
        assert st == dict(native=0, forwarded=2, analysis=0), st


def test_set_values_and_update_matrix_follow_the_closed_library():
    from cudalibrarysamples_b200 import cusparse_api as cs
    off, col = M.SR.stencil5_pattern(12)
    rows, nrhs = 144, 4
    v1 = M.values(rows, off, col, np.float64, seed=1)
    v2 = M.values(rows, off, col, np.float64, seed=2)
    dnew = np.random.default_rng(3).uniform(5, 6, rows)
    B = np.random.default_rng(4).uniform(-1, 1, rows * nrhs)
    res = {}
    for impl in ("b200", "cusparse"):
        api = cs.Api(impl)
        arr = dict(off=torch.tensor(off, device="cuda"), col=torch.tensor(col, device="cuda"), val=torch.tensor(v1, device="cuda"))
        other, dd = torch.tensor(v2, device="cuda"), torch.tensor(dnew, device="cuda")
        Bd, Cd = torch.tensor(B, device="cuda"), torch.zeros(rows * nrhs, dtype=torch.float64, device="cuda")
        s = cs.SpSMSolver(api, rows, arr, Bd, Cd, nrhs)
        out = [s().clone()]
        api.cusparseSpMatSetValues(s.mat, other)                 # after analysis: does not reach the solve
        out.append(s().clone())
        s.update(other, cs.CUSPARSE_SPSM_UPDATE_GENERAL)
        out.append(s().clone())
        s.update(dd, cs.CUSPARSE_SPSM_UPDATE_DIAGONAL)
        out.append(s().clone())
        torch.cuda.synchronize()
        s.close()
        res[impl] = [o.cpu().numpy() for o in out]
    for a, b in zip(res["b200"], res["cusparse"]):
        assert np.allclose(a, b, rtol=1e-12, atol=1e-12)
    assert np.array_equal(res["b200"][0], res["b200"][1]) and not np.allclose(res["b200"][1], res["b200"][2])


def test_c_aliasing_b_matches_the_closed_library():
    from cudalibrarysamples_b200 import cusparse_api as cs
    off, col = M.SR.stencil5_pattern(10)
    rows, nrhs = 100, 3
    val = M.values(rows, off, col, np.float64, seed=7)
    B = np.random.default_rng(8).uniform(-1, 1, rows * nrhs)
    res = {}
    for impl in ("b200", "cusparse"):
        api = cs.Api(impl)
        arr = dict(off=torch.tensor(off, device="cuda"), col=torch.tensor(col, device="cuda"), val=torch.tensor(val, device="cuda"))
        X = torch.tensor(B, device="cuda")
        s = cs.SpSMSolver(api, rows, arr, X, X, nrhs)
        s()
        torch.cuda.synchronize()
        s.close()
        res[impl] = X.cpu().numpy()
    assert np.allclose(res["b200"], res["cusparse"], rtol=1e-12, atol=1e-12)


def _forwarded(run):
    from cudalibrarysamples_b200 import cusparse_api as cs
    api = cs.Api("b200")
    api.reset_spsm_stats()
    run(api)
    torch.cuda.synchronize()
    return api.spsm_stats()


def test_forwarded_classes_are_counted_and_agree():
    from cudalibrarysamples_b200 import cusparse_api as cs
    off, col = M.SR.stencil5_pattern(8)
    rows, nrhs = 64, 4
    val = M.values(rows, off, col, np.float64, seed=9)
    B = np.random.default_rng(9).uniform(-1, 1, rows * nrhs)
    ref = shim_case("cusparse", rows, off, col, val, B, nrhs)
    # 64-bit indices
    out = {}

    def idx64(api):
        arr = dict(off=torch.tensor(off, dtype=torch.int64, device="cuda"), col=torch.tensor(col, dtype=torch.int64, device="cuda"),
                   val=torch.tensor(val, device="cuda"))
        out["c"] = cs.spsm(api, rows, arr, torch.tensor(B, device="cuda"), nrhs).cpu().numpy()
    st = _forwarded(idx64)
    assert st["native"] == 0 and st["forwarded"] >= 2 and np.allclose(out["c"], ref, rtol=1e-12, atol=1e-12)

    # a NON_UNIT matrix with a row that stores no diagonal: forwarded after the native analysis found it
    keep = ~((np.repeat(np.arange(rows), np.diff(off)) == 5) & (col == 5))
    off2 = np.concatenate([[0], np.cumsum(np.bincount(np.repeat(np.arange(rows), np.diff(off))[keep], minlength=rows))]).astype(np.int32)
    col2, val2 = col[keep], val[keep]

    def missing(api):
        arr = dict(off=torch.tensor(off2, device="cuda"), col=torch.tensor(col2, device="cuda"), val=torch.tensor(val2, device="cuda"))
        s = cs.SpSMSolver(api, rows, arr, torch.tensor(B, device="cuda"), torch.zeros(rows * nrhs, dtype=torch.float64, device="cuda"), nrhs)
        s()
        s.close()
    st = _forwarded(missing)
    assert st["forwarded"] >= 2, st

    # analysis under stream capture
    def captured(api):
        arr = dict(off=torch.tensor(off, device="cuda"), col=torch.tensor(col, device="cuda"), val=torch.tensor(val, device="cuda"))
        Bd, Cd = torch.tensor(B, device="cuda"), torch.zeros(rows * nrhs, dtype=torch.float64, device="cuda")
        h = api.cusparseCreate()
        mat = api.cusparseCreateCsr(rows, rows, int(col.size), arr["off"], arr["col"], arr["val"])
        matB = api.cusparseCreateDnMat(rows, nrhs, rows, Bd)
        matC = api.cusparseCreateDnMat(rows, nrhs, rows, Cd)
        d = api.cusparseSpSM_createDescr()
        size = api.cusparseSpSM_bufferSize(h, 0, 0, 1.0, mat, matB, matC, cs.CUDA_R_64F, 0, d)
        buf = torch.empty(max(size, 16), dtype=torch.uint8, device="cuda")
        s = torch.cuda.Stream()
        api.cusparseSetStream(h, s.cuda_stream)
        g = torch.cuda.CUDAGraph()
        try:
            with torch.cuda.graph(g, stream=s):
                api.cusparseSpSM_analysis(h, 0, 0, 1.0, mat, matB, matC, cs.CUDA_R_64F, 0, d, buf)
        except cs.CuSparseError:
            pass                                                 # whatever the closed library says under capture is its verdict
        torch.cuda.synchronize()
        api.cusparseSpSM_destroyDescr(d)
        api.cusparseDestroyDnMat(matB)
        api.cusparseDestroyDnMat(matC)
        api.cusparseDestroySpMat(mat)
        api.cusparseDestroy(h)
    st = _forwarded(captured)
    assert st["native"] == 0 and st["analysis"] == 0 and st["forwarded"] >= 1, st

    # batch count > 1 on B and C, and mixed types (fp32 A with fp64 B, C and compute): each step's status is the closed
    # library's, and the shim forwards (and counts) the analysis and the solve
    def batched(api):
        Bd, Cd = torch.tensor(np.tile(B, 2), device="cuda"), torch.zeros(2 * rows * nrhs, dtype=torch.float64, device="cuda")
        matB = api.cusparseCreateDnMat(rows, nrhs, rows, Bd)
        matC = api.cusparseCreateDnMat(rows, nrhs, rows, Cd)
        api.cusparseDnMatSetStridedBatch(matB, 2, rows * nrhs)
        api.cusparseDnMatSetStridedBatch(matC, 2, rows * nrhs)
        return raw_sequence(api, torch.tensor(val, device="cuda"), matB, matC, Bd, Cd)

    def mixed(api):
        Bd, Cd = torch.tensor(B, device="cuda"), torch.zeros(rows * nrhs, dtype=torch.float64, device="cuda")
        matB = api.cusparseCreateDnMat(rows, nrhs, rows, Bd)
        matC = api.cusparseCreateDnMat(rows, nrhs, rows, Cd)
        return raw_sequence(api, torch.tensor(val.astype(np.float32), device="cuda"), matB, matC, Bd, Cd)

    def raw_sequence(api, vald, matB, matC, Bd, Cd):
        """bufferSize, analysis (in a buffer of at least 1 MiB) and solve, fp64 compute: the three statuses and C."""
        offd, cold = torch.tensor(off, device="cuda"), torch.tensor(col, device="cuda")
        h = api.cusparseCreate()
        mat = api.cusparseCreateCsr(rows, rows, int(col.size), offd, cold, vald)
        d = api.cusparseSpSM_createDescr()
        one = C.c_double(1.0)
        pa = C.cast(C.pointer(one), C.c_void_p)
        size = C.c_size_t(0)
        s1 = api.lib.cusparseSpSM_bufferSize(h, 0, 0, pa, mat, matB, matC, cs.CUDA_R_64F, 0, d, C.byref(size))
        buf = torch.zeros(max(int(size.value), 1 << 20), dtype=torch.uint8, device="cuda")
        s2 = api.lib.cusparseSpSM_analysis(h, 0, 0, pa, mat, matB, matC, cs.CUDA_R_64F, 0, d, C.c_void_p(buf.data_ptr()))
        s3 = api.lib.cusparseSpSM_solve(h, 0, 0, pa, mat, matB, matC, cs.CUDA_R_64F, 0, d)
        torch.cuda.synchronize()
        out = (s1, s2, s3), Cd.cpu().numpy()
        api.cusparseSpSM_destroyDescr(d)
        api.cusparseDestroyDnMat(matB)
        api.cusparseDestroyDnMat(matC)
        api.cusparseDestroySpMat(mat)
        api.cusparseDestroy(h)
        return out

    for run in (batched, mixed):
        want, c_ref = run(cs.Api("cusparse"))
        res = {}
        st = _forwarded(lambda api: res.setdefault("r", run(api)))
        got, c_ours = res["r"]
        assert got == want, (run.__name__, got, want)
        assert st == dict(native=0, forwarded=2, analysis=0), (run.__name__, st)
        if want == (0, 0, 0):
            assert np.allclose(c_ours, c_ref, rtol=1e-12, atol=1e-12), run.__name__

    # COO A, and mixed types (fp32 A with fp64 dense matrices and compute): the closed library's status either way
    def coo(api):
        r = np.repeat(np.arange(rows), np.diff(off)).astype(np.int32)
        h = api.cusparseCreate()
        ro, co, vo = torch.tensor(r, device="cuda"), torch.tensor(col, device="cuda"), torch.tensor(val, device="cuda")
        mat = api.cusparseCreateCoo(rows, rows, int(col.size), ro, co, vo)
        Bd, Cd = torch.tensor(B, device="cuda"), torch.zeros(rows * nrhs, dtype=torch.float64, device="cuda")
        matB = api.cusparseCreateDnMat(rows, nrhs, rows, Bd)
        matC = api.cusparseCreateDnMat(rows, nrhs, rows, Cd)
        d = api.cusparseSpSM_createDescr()
        size = api.cusparseSpSM_bufferSize(h, 0, 0, 1.0, mat, matB, matC, cs.CUDA_R_64F, 0, d)
        buf = torch.empty(max(size, 16), dtype=torch.uint8, device="cuda")
        api.cusparseSpSM_analysis(h, 0, 0, 1.0, mat, matB, matC, cs.CUDA_R_64F, 0, d, buf)
        api.cusparseSpSM_solve(h, 0, 0, 1.0, mat, matB, matC, cs.CUDA_R_64F, 0, d)
        torch.cuda.synchronize()
        out["c"] = Cd.cpu().numpy()
        api.cusparseSpSM_destroyDescr(d)
        api.cusparseDestroyDnMat(matB)
        api.cusparseDestroyDnMat(matC)
        api.cusparseDestroySpMat(mat)
        api.cusparseDestroy(h)
    st = _forwarded(coo)
    assert st["native"] == 0 and st["forwarded"] >= 2 and np.allclose(out["c"], ref, rtol=1e-12, atol=1e-12)


def test_null_buffer_at_analysis_is_invalid_value():
    from cudalibrarysamples_b200 import cusparse_api as cs
    off, col = M.SR.stencil5_pattern(8)
    rows, nrhs = 64, 2
    val = M.values(rows, off, col, np.float64, seed=1)
    api = cs.Api("b200")
    api.reset_spsm_stats()
    arr = dict(off=torch.tensor(off, device="cuda"), col=torch.tensor(col, device="cuda"), val=torch.tensor(val, device="cuda"))
    Bd, Cd = torch.rand(rows * nrhs, dtype=torch.float64, device="cuda"), torch.zeros(rows * nrhs, dtype=torch.float64, device="cuda")
    with pytest.raises(cs.CuSparseError) as e:
        cs.SpSMSolver(api, rows, arr, Bd, Cd, nrhs, buffer=None)
    assert e.value.status == cs.CUSPARSE_STATUS_INVALID_VALUE
    assert api.spsm_stats()["forwarded"] == 0


def test_reference_sample_passes_on_the_shim():
    exe = os.path.join(ROOT, "oracle", "_ref", "spsm_csr_example.b200")
    if not os.path.exists(exe):
        pytest.skip("oracle/_ref not built (needs the reference checkout)")
    env = dict(os.environ, B200SPMV_LOG="1")
    env.pop("B200SPMV_CUSPARSE", None)
    p = subprocess.run([exe], env=env, capture_output=True, text=True, timeout=120)
    assert "spsm_csr_example test PASSED" in p.stdout, p.stdout + p.stderr
