"""GPU: the native SDDMM of libb200spmv.so (cusparseSDDMM_*, b200sddmm_csr) bit for bit against the int64 reference of
oracle/sddmm_ref.py over every layout, K edge, chunk border, scalar mode and batch layout; against the closed library within the
dot-product error bound; status parity; repeatability and graph replay; forwarded kinds; the two reference samples."""
import ctypes as C
import itertools
import os
import subprocess

import numpy as np
import pytest
import torch

from cudalibrarysamples_b200 import cusparse_api as cs
from cudalibrarysamples_b200 import lib as _lib
from oracle import exact as X
from oracle import oracle as O
from oracle import sddmm_ref as R

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEV = torch.device("cuda:0")
NT, TR = cs.CUSPARSE_OPERATION_NON_TRANSPOSE, cs.CUSPARSE_OPERATION_TRANSPOSE
ROW, COL = cs.CUSPARSE_ORDER_ROW, cs.CUSPARSE_ORDER_COL
TD = {np.float32: torch.float32, np.float64: torch.float64}
LAYOUTS = list(itertools.product((NT, TR), (ROW, COL), (NT, TR), (ROW, COL)))      # opA, order A, opB, order B


def P():
    return R.params()


def store(X_, op, order, dt, pad=0, shift=0):
    """The buffer (a view `shift` elements into its allocation, NaN in every unused slot) and ld of a dense operand whose op() is
    X_ (float array, NaN allowed)."""
    S = X_ if op == NT else X_.T
    r, c = S.shape
    if order == ROW:
        ld = max(c + pad, 1)
        buf = np.full(shift + r * ld + 1, np.nan, dt)
        buf[shift:shift + r * ld].reshape(r, ld)[:, :c] = S
    else:
        ld = max(r + pad, 1)
        buf = np.full(shift + c * ld + 1, np.nan, dt)
        buf[shift:shift + c * ld].reshape(c, ld)[:, :r] = S.T
    t = torch.tensor(buf, device=DEV)
    return t[shift:], ld


def structure(lens, n, seed, base=0):
    off, col = X.lens_to_structure(np.asarray(lens, np.int64), n, seed)
    return (off + base).astype(np.int32), (col + base).astype(np.int32)


def guarded(c0, dt):
    """C's values as a view with NaN guard elements on both sides; returns (view, whole buffer)"""
    buf = torch.full((c0.size + 8,), float("nan"), dtype=TD[dt], device=DEV)
    buf[4:4 + c0.size] = torch.tensor(c0.astype(dt), device=DEV)
    return buf[4:4 + c0.size], buf


def strides(layout, lda, ldb):
    """(sai, sak, sbk, sbj) of b200sddmm_csr for a layout (opA, order A, opB, order B) with these leading dimensions"""
    opA, oa, opB, ob = layout
    ar, ac = (lda, 1) if oa == ROW else (1, lda)                   # element (r, c) of the stored matrix: r * ar + c * ac
    br, bc = (ldb, 1) if ob == ROW else (1, ldb)
    sai, sak = (ac, ar) if opA == TR else (ar, ac)
    sbk, sbj = (bc, br) if opB == TR else (br, bc)
    return sai, sak, sbk, sbj


def shim_native(dt, k, sbk):
    """the route's measured rule (DESIGN.md 3.13): fp32 with K <= 32 or with an op(B) that is not K-contiguous"""
    return dt == np.float32 and (k <= 32 or (k > 1 and sbk != 1))


def layer2(dt, m, n, k, off, col, val, base, alpha, beta, A, st, B, batch=1, off_stride=0, cv_stride=0, a_stride=0, b_stride=0,
           buffer=True):
    """b200sddmm_csr directly (every layout); alpha / beta: numbers (host) or device tensors"""
    lib = _lib.shim()
    sai, sak, sbk, sbj = st
    i64 = C.c_int64
    need = lib.b200sddmm_csr_workspace_bytes(int(dt == np.float64), i64(m), i64(n), i64(k), i64(sai), i64(sak), i64(sbk), i64(sbj),
                                             batch, i64(a_stride), i64(b_stride))
    ws = torch.empty(max(need, 16), dtype=torch.uint8, device=DEV) if buffer else None
    dev = isinstance(alpha, torch.Tensor)
    ct = C.c_float if dt == np.float32 else C.c_double
    pa, pb = (C.c_void_p(alpha.data_ptr()), C.c_void_p(beta.data_ptr())) if dev else (C.byref(ct(alpha)), C.byref(ct(beta)))
    rc = lib.b200sddmm_csr(C.c_void_p(torch.cuda.current_stream().cuda_stream), int(dt == np.float64), i64(m), i64(n), i64(k),
                           i64(len(col) // batch), C.c_void_p(off.data_ptr()), C.c_void_p(col.data_ptr()), C.c_void_p(val.data_ptr()), base,
                           pa, pb, int(dev), C.c_void_p(A.data_ptr()), i64(sai), i64(sak), C.c_void_p(B.data_ptr()), i64(sbk), i64(sbj),
                           batch, i64(off_stride), i64(cv_stride), i64(a_stride), i64(b_stride),
                           C.c_void_p(ws.data_ptr() if ws is not None else 0), C.c_size_t(need if buffer else 0))
    assert rc == 0
    torch.cuda.synchronize()


def run_case(kind, off, col, m, n, k, layout=(NT, ROW, TR, ROW), alpha=1.0, beta=0.0, base=0, device_scalars=False, pad=0, shift=0,
             buffer="auto", nan_unused=True, seed=1):
    """the same exact product through b200sddmm_csr and, where the route keeps it native, through cusparseSDDMM; asserts bit
    equality with the int64 reference, untouched guards, and forwarded == 0 on the shim"""
    opA, oa, opB, ob = layout
    dt = R.NP_T[kind]
    nnz = len(col)
    a, b, c0 = R.values(kind, m, n, k, nnz, seed)
    R.check_exact(off, col, a, b, c0, alpha, beta, R.MANTISSA[kind], base)
    af, bf = a.astype(dt), b.astype(dt)
    if nan_unused:                                   # rows of A / columns of B that C never references hold NaN
        used_r = np.zeros(m, bool)
        used_r[R.rows_of(off, base)] = True
        used_c = np.zeros(n, bool)
        used_c[np.asarray(col, np.int64) - base] = True
        af[~used_r] = np.nan
        bf[:, ~used_c] = np.nan
    A, lda = store(af, opA, oa, dt, pad, shift)
    B, ldb = store(bf, opB, ob, dt, pad, shift)
    st = strides(layout, lda, ldb)
    ref = R.reference(off, col, a, b, c0, alpha, beta, base).astype(dt)
    al, be = alpha, beta
    if device_scalars:
        al, be = torch.tensor([alpha], dtype=TD[dt], device=DEV), torch.tensor([beta], dtype=TD[dt], device=DEV)
    offt, colt = torch.tensor(off, device=DEV), torch.tensor(col, device=DEV)
    for via in ("layer2", "shim"):
        if via == "shim" and not shim_native(dt, k, st[2]):
            continue
        cv, whole = guarded(np.full(nnz, np.nan) if beta == 0 else c0, dt)
        if via == "layer2":
            layer2(dt, m, n, k, offt, colt, cv, base, al, be, A, st, B, buffer=buffer is not None)
        else:
            api = cs.Api("b200")
            api.reset_stats()
            cs.sddmm(api, m, n, k, A, B, dict(off=offt, col=colt, val=cv, nnz=nnz), alpha=al, beta=be, opA=opA, opB=opB, order_a=oa,
                     order_b=ob, lda=lda, ldb=ldb, base=base, buffer=buffer)
            assert api.stats()["forwarded"] == 0 and api.stats()["native"] == 1, api.stats()
        got = cv.cpu().numpy()
        assert np.array_equal(got, ref), (via, kind, layout, k, np.flatnonzero(got != ref)[:10])
        g = whole.cpu().numpy()
        assert np.isnan(g[:4]).all() and np.isnan(g[-4:]).all()


# ---------------------------------------------------------------------------------------------- exact sweeps
@pytest.mark.parametrize("layout", LAYOUTS, ids=lambda l: "A%s%s_B%s%s" % ("nt"[l[0]], "?cr"[l[1]], "nt"[l[2]], "?cr"[l[3]]))
@pytest.mark.parametrize("kind", ["f32", "f64", "wide"])
@pytest.mark.parametrize("k", [7, 64])
@pytest.mark.parametrize("buffer", ["auto", None])
def test_every_layout_exact(layout, kind, k, buffer):
    m, n = 70, 90
    lens = [0, 3, 40, 0, 1] + [5] * 60 + [0] * 5
    off, col = structure(lens, n - 10, 3)                         # the last 10 columns of B are never referenced
    run_case(kind, off, col, m, n, k, layout=layout, buffer=buffer, pad=3 if k == 7 else 0)


@pytest.mark.parametrize("kind", ["f32", "f64", "wide"])
@pytest.mark.parametrize("layout", [(NT, ROW, TR, ROW), (NT, ROW, NT, ROW)], ids=["kcontig", "sample"])
def test_k_edges_exact(kind, layout):
    p = P()
    dt = R.NP_T[kind]
    off, col = structure([2, 0, 33, 1, 7, 0, 64, 3], 70, 4)
    for k in [k for k in R.k_edges(p, np.dtype(dt).itemsize) if k > 0]:       # K = 0: test_k_zero
        for buffer in ("auto", None):
            run_case(kind, off, col, 8, 70, k, layout=layout, buffer=buffer, alpha=-2.0, beta=0.5)


@pytest.mark.parametrize("base", [0, 1])
@pytest.mark.parametrize("scal", R.SCALARS)
@pytest.mark.parametrize("device_scalars", [False, True])
@pytest.mark.parametrize("kind", ["f32", "wide"])
def test_scalars_base_and_pointer_mode(base, scal, device_scalars, kind):
    off, col = structure([4, 0, 9, 1, 17], 40, 5, base)
    run_case(kind, off, col, 5, 40, 24, alpha=scal[0], beta=scal[1], base=base, device_scalars=device_scalars)


def test_chunk_borders_exact():
    """row ends at every warp-chunk border +-1, empty rows, and one row longer than several chunks"""
    p = P()
    w = p["warp_chunk"]
    lens, pos = [], 0
    for target in (w - 1, w, w + 1, 2 * w - 1, 2 * w + 1, 3 * w):
        if target > pos:
            lens.append(target - pos)
            pos = target
        lens.append(0)
    lens += [5 * w + 3, 0, 0, 1, w, 1]
    n = max(lens) + 5
    off, col = structure(lens, n, 6)
    for kind, k in (("f32", 1), ("f32", 64), ("f64", 3), ("wide", 130)):
        for layout in ((NT, ROW, TR, ROW), (TR, COL, NT, ROW)):
            run_case(kind, off, col, len(lens), n, k, layout=layout, alpha=0.5, beta=-1.0)


@pytest.mark.parametrize("kind", ["f32", "f64"])
def test_padding_misaligned_views_and_nan(kind):
    off, col = structure([3, 0, 12, 8, 1, 0], 30, 7)
    for layout in LAYOUTS[::3]:
        for shift, pad in ((1, 0), (1, 5), (0, 4)):
            for buffer in ("auto", None):
                run_case(kind, off, col, 6, 30, 40, layout=layout, shift=shift, pad=pad, buffer=buffer)


def test_misaligned_and_small_buffers_take_the_strided_path():
    """layer 2 directly: the sample's layout with a misaligned and with a too small workspace gives the same bits"""
    lib = _lib.shim()
    off, col = structure([3, 7, 0, 20], 33, 8)
    m, n, k = 4, 33, 40
    a, b, c0 = R.values("f32", m, n, k, len(col), 9)
    ref = R.reference(off, col, a, b, c0, 1.0, 0.0).astype(np.float32)
    A = torch.tensor(a.astype(np.float32).ravel(), device=DEV)
    B = torch.tensor(b.astype(np.float32).ravel(), device=DEV)             # k x n row-major: sbk = n, sbj = 1
    need = lib.b200sddmm_csr_workspace_bytes(0, C.c_int64(m), C.c_int64(n), C.c_int64(k), C.c_int64(k), C.c_int64(1), C.c_int64(n),
                                             C.c_int64(1), 1, C.c_int64(0), C.c_int64(0))
    assert need >= n * k * 4
    ws = torch.zeros(need + 64, dtype=torch.uint8, device=DEV)
    offt, colt = torch.tensor(off, device=DEV), torch.tensor(col, device=DEV)
    al, be = C.c_float(1.0), C.c_float(0.0)
    for wp, wb in ((ws.data_ptr(), need), (ws.data_ptr() + 4, need), (ws.data_ptr(), need - 256), (0, 0)):
        val = torch.full((len(col),), float("nan"), device=DEV)
        rc = lib.b200sddmm_csr(C.c_void_p(torch.cuda.current_stream().cuda_stream), 0, C.c_int64(m), C.c_int64(n), C.c_int64(k),
                               C.c_int64(len(col)), C.c_void_p(offt.data_ptr()), C.c_void_p(colt.data_ptr()), C.c_void_p(val.data_ptr()),
                               0, C.byref(al), C.byref(be), 0, C.c_void_p(A.data_ptr()), C.c_int64(k), C.c_int64(1),
                               C.c_void_p(B.data_ptr()), C.c_int64(n), C.c_int64(1), 1, C.c_int64(0), C.c_int64(0), C.c_int64(0),
                               C.c_int64(0), C.c_void_p(wp), C.c_size_t(wb))
        assert rc == 0
        torch.cuda.synchronize()
        assert np.array_equal(val.cpu().numpy(), ref)


def test_k_zero_scales_c_by_beta():
    """K = 0 through layer 2: C = beta * C, A and B never read (NULL)"""
    lib = _lib.shim()
    off, col = structure([3, 0, 5], 9, 10)
    for dt, ct, be in ((np.float32, C.c_float, 0.5), (np.float64, C.c_double, 0.0)):
        c0 = np.arange(len(col), dtype=dt) * 2
        val = torch.tensor(c0 if be else np.full(len(col), np.nan, dt), device=DEV)
        offt, colt = torch.tensor(off, device=DEV), torch.tensor(col, device=DEV)
        al, bb = ct(-2.0), ct(be)
        rc = lib.b200sddmm_csr(C.c_void_p(torch.cuda.current_stream().cuda_stream), int(dt == np.float64), C.c_int64(3), C.c_int64(9),
                               C.c_int64(0), C.c_int64(len(col)), C.c_void_p(offt.data_ptr()), C.c_void_p(colt.data_ptr()),
                               C.c_void_p(val.data_ptr()), 0, C.byref(al), C.byref(bb), 0, None, C.c_int64(0), C.c_int64(0), None,
                               C.c_int64(0), C.c_int64(0), 1, C.c_int64(0), C.c_int64(0), C.c_int64(0), C.c_int64(0), None, C.c_size_t(0))
        assert rc == 0
        torch.cuda.synchronize()
        assert np.array_equal(val.cpu().numpy(), (be * c0).astype(dt))


# ---------------------------------------------------------------------------------------------- batches
@pytest.mark.parametrize("kind", ["f32", "wide"])
@pytest.mark.parametrize("shared", ["none", "offsets", "A", "B"])
@pytest.mark.parametrize("layout", [(NT, ROW, NT, ROW), (NT, ROW, TR, ROW), (TR, COL, NT, COL)], ids=["sample", "kcontig", "colmajor"])
def test_strided_batches_exact(kind, shared, layout):
    opA, oa, opB, ob = layout
    dt = R.NP_T[kind]
    nb, m, n, k = 3, 9, 21, 20
    lens = [2, 0, 5, 1, 7, 0, 3, 9, 4]
    pats = [structure(lens, n, 20 + i) for i in range(nb)]
    off = pats[0][0]
    col_all = np.concatenate([p[1] for p in pats])                # same row lengths: the offsets can be shared
    nnz = len(pats[0][1])
    vals = [R.values(kind, m, n, k, nnz, 30 + i) for i in range(nb)]
    if shared == "A":
        vals = [(vals[0][0],) + v[1:] for v in vals]
    if shared == "B":
        vals = [(v[0], vals[0][1], v[2]) for v in vals]
    As = [store(v[0].astype(dt), opA, oa, dt)[0] for v in (vals[:1] if shared == "A" else vals)]
    Bs = [store(v[1].astype(dt), opB, ob, dt)[0] for v in (vals[:1] if shared == "B" else vals)]
    _, lda = store(vals[0][0].astype(dt), opA, oa, dt)
    _, ldb = store(vals[0][1].astype(dt), opB, ob, dt)
    a_size, b_size = As[0].numel(), Bs[0].numel()
    A, B = torch.cat(As), torch.cat(Bs)
    c0 = np.concatenate([v[2] for v in vals])
    if shared == "offsets":
        off_t, off_stride = torch.tensor(off, device=DEV), 0
    else:
        off_t, off_stride = torch.tensor(np.concatenate([off] * nb), device=DEV), len(off)
    colt = torch.tensor(col_all, device=DEV)
    a_stride, b_stride = 0 if shared == "A" else a_size, 0 if shared == "B" else b_size
    st = strides(layout, lda, ldb)
    for via in ("layer2", "shim"):
        if via == "shim" and not shim_native(dt, k, st[2]):
            continue
        cv = torch.tensor(c0.astype(dt), device=DEV)
        if via == "layer2":
            layer2(dt, m, n, k, off_t, colt, cv, 0, -2.0, 0.5, A, st, B, batch=nb, off_stride=off_stride, cv_stride=nnz, a_stride=a_stride,
                   b_stride=b_stride)
        else:
            api = cs.Api("b200")
            api.reset_stats()
            cs.sddmm_batched(api, nb, m, n, k, A, B, dict(off=off_t, col=colt, val=cv, nnz=nnz), alpha=-2.0, beta=0.5, opA=opA, opB=opB,
                             order_a=oa, order_b=ob, lda=lda, ldb=ldb, off_stride=off_stride, a_stride=a_stride, b_stride=b_stride)
            assert api.stats()["forwarded"] == 0 and api.stats()["native"] == 1
        got = cv.cpu().numpy()
        for i in range(nb):
            a, b, c = vals[i]
            ref = R.reference(off, pats[i][1], a, b, c, -2.0, 0.5).astype(dt)
            assert np.array_equal(got[i * nnz:(i + 1) * nnz], ref), (via, i)


def test_batched_sample_toy():
    S = R.samples()["sddmm_csr_batched"]
    api = cs.Api("b200")
    api.reset_stats()
    val = torch.zeros(18, device=DEV)
    A = torch.tensor(np.ravel(S["A"]), dtype=torch.float32, device=DEV)
    B = torch.tensor(np.ravel(S["B"]), dtype=torch.float32, device=DEV)
    cs.sddmm_batched(api, 2, 4, 3, 4, A, B, dict(off=torch.tensor(S["off"], dtype=torch.int32, device=DEV),
                                                col=torch.tensor(np.ravel(S["col"]), dtype=torch.int32, device=DEV), val=val, nnz=9))
    assert np.array_equal(val.cpu().numpy(), np.ravel(S["C_result"]))
    assert api.stats()["forwarded"] == 0


# ---------------------------------------------------------------------------------------------- the closed library
def random_case(pattern, k, seed):
    off, col = pattern
    m = len(off) - 1
    n = int(col.max()) + 1 if len(col) else 1
    rng = np.random.default_rng(seed)
    a = rng.uniform(-1, 1, (m, k))
    b = rng.uniform(-1, 1, (k, n))
    return off, col, m, n, a, b


@pytest.mark.parametrize("pattern", ["rmat", "stencil"])
@pytest.mark.parametrize("dt", [np.float32, np.float64])
@pytest.mark.parametrize("layout", [(NT, ROW, TR, ROW), (NT, ROW, NT, ROW), (TR, COL, NT, COL), (NT, COL, TR, COL)],
                         ids=["kcontig", "sample", "colmajor", "mixed"])
def test_parity_with_the_closed_library(pattern, dt, layout):
    if pattern == "rmat":
        off, col, _ = O.rmat_csr(4096, avg_nnz=16, seed=11, val_seed=12)
    else:
        off, col, _ = R_stencil(64)
    k = 48
    off, col, m, n, a, b = random_case((off, col), k, 13)
    opA, oa, opB, ob = layout
    A, lda = store(a.astype(dt), opA, oa, dt)
    B, ldb = store(b.astype(dt), opB, ob, dt)
    ref = np.einsum("ek,ek->e", a[R.rows_of(off)], b[:, col].T)
    bound = k * np.finfo(dt).eps / 2 * np.einsum("ek,ek->e", np.abs(a[R.rows_of(off)]), np.abs(b[:, col].T))
    res = {}
    offt, colt = torch.tensor(off, device=DEV), torch.tensor(col, device=DEV)
    for impl in ("b200", "cusparse"):                              # ours through layer 2: every layout, also those the route forwards
        cv = torch.zeros(len(col), dtype=TD[dt], device=DEV)
        try:
            if impl == "b200":
                layer2(dt, m, n, k, offt, colt, cv, 0, 1.0, 0.0, A, strides(layout, lda, ldb), B)
            else:
                cs.sddmm(cs.Api(impl), m, n, k, A, B, dict(off=offt, col=colt, val=cv), opA=opA, opB=opB, order_a=oa, order_b=ob,
                         lda=lda, ldb=ldb)
            res[impl] = cv.cpu().numpy().astype(np.float64)
        except cs.CuSparseError as e:
            assert impl == "cusparse", e
            res[impl] = None                                       # the closed library rejects this combination: reference only
    for impl, got in res.items():
        if got is not None:
            assert (np.abs(got - ref) <= bound + 1e-300).all(), impl


def R_stencil(g):
    from oracle import spsv_ref as SR
    off, col = SR.stencil5_pattern(g)
    return off, col, None


def test_status_parity_for_shape_mismatches():
    """each mismatch: the same status from both libraries at bufferSize and at the call"""
    off = torch.tensor([0, 1, 2, 3, 4], dtype=torch.int32, device=DEV)
    col = torch.tensor([0, 1, 2, 0], dtype=torch.int32, device=DEV)
    buf = torch.zeros(1 << 16, dtype=torch.uint8, device=DEV)
    X_ = torch.zeros(4096, device=DEV)
    cases = {  # (A rows, A cols, opA, B rows, B cols, opB) for C 4 x 3
        "ok": (4, 5, NT, 5, 3, NT), "a_rows": (3, 5, NT, 5, 3, NT), "k_mismatch": (4, 5, NT, 6, 3, NT),
        "b_cols": (4, 5, NT, 5, 4, NT), "a_transposed_wrong": (4, 5, TR, 5, 3, NT), "b_transposed_wrong": (4, 5, NT, 5, 3, TR),
        "both_transposed_ok": (5, 4, TR, 3, 5, TR)}
    for name, (ar, ac, opA, br, bc, opB) in cases.items():
        out = {}
        for impl in ("b200", "cusparse"):
            api = cs.Api(impl)
            h = api.cusparseCreate()
            matA = api.cusparseCreateDnMat(ar, ac, ac, X_, ROW)
            matB = api.cusparseCreateDnMat(br, bc, bc, X_, ROW)
            val = torch.zeros(4, device=DEV)
            matC = api.cusparseCreateCsr(4, 3, 4, off, col, val)
            st = []
            for fn, extra in (("cusparseSDDMM_bufferSize", C.byref(C.c_size_t(0))), ("cusparseSDDMM", C.c_void_p(buf.data_ptr()))):
                one, zero = C.c_float(1.0), C.c_float(0.0)
                st.append(getattr(api.lib, fn)(h, opA, opB, C.byref(one), matA, matB, C.byref(zero), matC, cs.CUDA_R_32F, 0, extra))
            torch.cuda.synchronize()
            api.cusparseDestroyDnMat(matA)
            api.cusparseDestroyDnMat(matB)
            api.cusparseDestroySpMat(matC)
            api.cusparseDestroy(h)
            out[impl] = st
        assert out["b200"] == out["cusparse"], (name, out)


# ---------------------------------------------------------------------------------------------- repeatability and graphs
def test_repeated_calls_and_graph_replay_give_identical_bits():
    off, col, _ = O.rmat_csr(8192, avg_nnz=16, seed=21, val_seed=22)
    m = n = 8192
    k = 64
    rng = np.random.default_rng(23)
    A = torch.tensor(rng.uniform(-1, 1, m * k).astype(np.float32), device=DEV)
    Bt = torch.tensor(rng.uniform(-1, 1, n * k).astype(np.float32), device=DEV)      # opB = TRANSPOSE, row-major N x K
    Bs = Bt.view(n, k).t().contiguous().view(-1)                                       # the sample's layout (K x N row-major)
    offt, colt = torch.tensor(off, device=DEV), torch.tensor(col, device=DEV)
    lib = _lib.shim()
    al, be = C.c_float(1.5), C.c_float(0.0)
    for B, sbk, sbj in ((Bt, 1, k), (Bs, n, 1)):
        need = lib.b200sddmm_csr_workspace_bytes(0, C.c_int64(m), C.c_int64(n), C.c_int64(k), C.c_int64(k), C.c_int64(1), C.c_int64(sbk),
                                                 C.c_int64(sbj), 1, C.c_int64(0), C.c_int64(0))
        ws = torch.empty(max(need, 16), dtype=torch.uint8, device=DEV)
        val = torch.empty(len(col), device=DEV)

        def call():
            return lib.b200sddmm_csr(C.c_void_p(torch.cuda.current_stream().cuda_stream), 0, C.c_int64(m), C.c_int64(n), C.c_int64(k),
                                     C.c_int64(len(col)), C.c_void_p(offt.data_ptr()), C.c_void_p(colt.data_ptr()),
                                     C.c_void_p(val.data_ptr()), 0, C.byref(al), C.byref(be), 0, C.c_void_p(A.data_ptr()), C.c_int64(k),
                                     C.c_int64(1), C.c_void_p(B.data_ptr()), C.c_int64(sbk), C.c_int64(sbj), 1, C.c_int64(0),
                                     C.c_int64(0), C.c_int64(0), C.c_int64(0), C.c_void_p(ws.data_ptr()), C.c_size_t(need))
        assert call() == 0
        torch.cuda.synchronize()
        first = val.clone()
        for _ in range(3):
            assert call() == 0
        torch.cuda.synchronize()
        assert torch.equal(val, first)
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        g = torch.cuda.CUDAGraph()
        with torch.cuda.stream(s):
            with torch.cuda.graph(g, stream=s):
                assert call() == 0
        val.fill_(float("nan"))
        for _ in range(3):
            g.replay()
        torch.cuda.synchronize()
        assert torch.equal(val, first)


# ---------------------------------------------------------------------------------------------- forwarded kinds
def test_forwarded_kinds_are_counted():
    off32 = torch.tensor([0, 1, 2, 3, 4], dtype=torch.int32, device=DEV)
    col32 = torch.tensor([0, 1, 2, 0], dtype=torch.int32, device=DEV)
    X_ = torch.ones(64, device=DEV)
    api = cs.Api("b200")

    def once(off, col, val, opA=NT, opB=NT, ct=cs.CUDA_R_32F, a_batch=1, c_batch=1, k=5, X_=X_):
        h = api.cusparseCreate()
        matA = api.cusparseCreateDnMat(4, k, k, X_, ROW)
        matB = api.cusparseCreateDnMat(k, 3, 3, X_, ROW) if opB == NT else api.cusparseCreateDnMat(3, k, k, X_, ROW)
        if a_batch > 1:
            api.cusparseDnMatSetStridedBatch(matA, a_batch, 20)
        matC = api.cusparseCreateCsr(4, 3, 4, off, col, val)
        if c_batch > 1:
            api.cusparseCsrSetStridedBatch(matC, c_batch, 0, 4)
        api.reset_stats()
        ctype = C.c_double if ct == cs.CUDA_R_64F else C.c_float
        one, zero = ctype(1.0), ctype(0.0)
        buf = torch.zeros(1 << 20, dtype=torch.uint8, device=DEV)
        api.lib.cusparseSDDMM(h, opA, opB, C.byref(one), matA, matB, C.byref(zero), matC, ct, 0, C.c_void_p(buf.data_ptr()))
        torch.cuda.synchronize()
        st = api.stats()
        api.cusparseDestroyDnMat(matA)
        api.cusparseDestroyDnMat(matB)
        api.cusparseDestroySpMat(matC)
        api.cusparseDestroy(h)
        return st

    val = torch.zeros(16, device=DEV)
    assert once(off32, col32, val) == dict(native=1, forwarded=0, analyze=0)
    assert once(off32.long(), col32.long(), val)["forwarded"] == 1                      # 64-bit indices
    assert once(off32, col32, val, opA=cs.CUSPARSE_OPERATION_CONJUGATE_TRANSPOSE)["forwarded"] == 1
    assert once(off32, col32, val, ct=cs.CUDA_R_64F)["forwarded"] == 1                  # compute type != value type
    assert once(off32, col32, val, a_batch=3, c_batch=2)["forwarded"] == 1              # 3 matrices of A for 2 of C
    big = torch.ones(1024, device=DEV)
    assert once(off32, col32, val, k=64, X_=big) == dict(native=1, forwarded=0, analyze=0)       # the sample's layout at K = 64
    assert once(off32, col32, val, k=64, opB=TR, X_=big)["forwarded"] == 1                       # K-contiguous, K > 32: slower here
    d64 = torch.ones(1024, dtype=torch.float64, device=DEV)
    assert once(off32, col32, torch.zeros(16, dtype=torch.float64, device=DEV), ct=cs.CUDA_R_64F, X_=d64)["forwarded"] == 1   # fp64


# ---------------------------------------------------------------------------------------------- the reference samples
@pytest.mark.parametrize("name", ["sddmm_csr", "sddmm_csr_batched"])
def test_reference_sample_runs_natively(name):
    exe = os.path.join(ROOT, "oracle", "_ref", f"{name}_example.b200")
    if not os.path.exists(exe):
        pytest.skip("oracle/_ref not built")
    env = {k: v for k, v in os.environ.items() if not k.startswith("B200SPMV_")}
    env["B200SPMV_LOG"] = "1"
    p = subprocess.run([exe], capture_output=True, text=True, timeout=120, env=env)
    assert p.returncode == 0, p.stdout + p.stderr
    assert f"{name}_example test PASSED" in p.stdout
    assert "[b200spmv] SDDMM" in p.stderr and "forwarded" not in p.stderr, p.stderr
