"""The hot-column part of the flat CSR plan (b200spmv_csr_flat_hot_analyze in cudalibrarysamples_b200/csrc/spmv_csr_flat.cu).

Preprocess picks the most-used columns of x that fit a byte budget, numbers them in ascending column order, and writes colp
(~slot for a hot column, else the 0-based column).  Every SpMV with H > 0 packs x[hot[j]] densely and csr_flat_kernel reads
colp: the same products in the same order, so y must be bit-identical to the call that reads col_ind.

hot_plan() below restates the plan in numpy; the GPU tests compare the device plan with it bit for bit and compare the
products of both paths with torch.equal (and with the exact integer reference on the exact-arithmetic profiles)."""
import ctypes as C

import numpy as np
import pytest

from oracle import exact as E
from oracle import oracle as O

PLAN_PAD = 2048          # the flat plan pads nnz to whole CTAs of 2048 non-zeros


def hot_plan(col, base, cols, hot_bytes, value_bytes, min_permille, bins):
    """numpy restatement: (hot columns ascending, tau, colp padded to PLAN_PAD).  tau = 0 and no colp when there is no hot plan."""
    nnz = col.size
    npad = (nnz + PLAN_PAD - 1) // PLAN_PAD * PLAN_PAD
    if hot_bytes == 0 or nnz == 0 or cols > npad:
        return np.zeros(0, np.int32), 0, None
    c = np.asarray(col, np.int64) - base
    cnt = np.bincount(c, minlength=cols)
    slots = hot_bytes // value_bytes
    hist = np.bincount(np.minimum(cnt[cnt >= 2], bins - 1), minlength=bins)
    h, tau = 0, 0
    for t in range(bins - 1, 1, -1):                 # the smallest tau >= 2 whose columns fit the slots
        if h + hist[t] > slots:
            break
        h += int(hist[t])
        tau = t
    hot = np.nonzero(cnt >= tau)[0] if tau else np.zeros(0, np.int64)
    if tau == 0 or h == 0 or int(cnt[hot].sum()) * 1000 < min_permille * nnz:
        return np.zeros(0, np.int32), 0, None
    slot = np.full(cols, -1, np.int64)
    slot[hot] = np.arange(hot.size)
    colp = np.zeros(npad, np.int64)
    colp[:nnz] = np.where(slot[c] >= 0, ~slot[c], c)
    return hot.astype(np.int32), tau, colp.astype(np.int32)


def skewed_cols(rows, cols, per_row, seed):
    """CSR whose columns are drawn from a Zipf-like law: a few columns take most of the non-zeros."""
    rng = np.random.default_rng(seed)
    w = 1.0 / np.arange(1, cols + 1) ** 1.1
    perm = rng.permutation(cols)
    lens, parts = [], []
    for l in rng.integers(0, 2 * per_row, rows):
        r = np.unique(perm[rng.choice(cols, size=int(l), p=w / w.sum())])       # sorted, duplicates merged
        lens.append(r.size)
        parts.append(r)
    off = np.concatenate([[0], np.cumsum(lens)]).astype(np.int32)
    return off, np.concatenate(parts).astype(np.int32)


def test_hot_plan_reference_invariants():
    """The restatement on an R-MAT matrix: hot columns fit the budget, every hot column is used at least tau times and no cold one
    is, tau - 1 would not fit, colp decodes back to col_ind, and the padding is a column that is never hot."""
    off, col, _ = O.rmat_csr(50000, avg_nnz=16, seed=7, val_seed=8)
    cols = off.size - 1
    hot, tau, colp = hot_plan(col, 0, cols, 128 * 1024, 8, 200, 1 << 16)
    cnt = np.bincount(col, minlength=cols)
    assert tau >= 2 and 0 < hot.size <= 128 * 1024 // 8
    assert np.all(np.diff(hot) > 0)
    assert np.all(cnt[hot] >= tau) and np.count_nonzero(cnt >= tau) == hot.size
    assert tau == 2 or np.count_nonzero(cnt >= tau - 1) > 128 * 1024 // 8
    assert int(cnt[hot].sum()) * 5 >= col.size
    cp = colp[:col.size]
    assert np.array_equal(np.where(cp < 0, hot[np.where(cp < 0, ~cp, 0)], cp), col)
    assert np.all(colp[col.size:] == 0) and colp.size % PLAN_PAD == 0
    # a matrix whose columns are all used equally often, and more of them than the budget holds, has none worth packing
    g = O.gen_stencil5(300)
    assert hot_plan(g[1], 0, g[0].size - 1, 128 * 1024, 8, 200, 1 << 16)[1] == 0


# ------------------------------------------------------------------------------------------------------------------ GPU
def _lib():
    from cudalibrarysamples_b200 import lib
    L = lib.shim()
    L.b200spmv_csr_flat_workspace_bytes.restype = C.c_size_t
    return L


def _params(L):
    hb, mp, nb = C.c_int32(), C.c_int32(), C.c_int32()
    L.b200spmv_csr_flat_hot_params(C.byref(hb), C.byref(mp), C.byref(nb))
    return hb.value, mp.value, nb.value


def _analyze(L, torch, off, col, base, cols, dtype):
    """flat plan + hot plan in a workspace pre-filled with garbage; returns (workspace, H)"""
    rows, nnz = off.size - 1, col.size
    ws = torch.full((L.b200spmv_csr_flat_workspace_bytes(C.c_int64(rows), C.c_int64(nnz)),), 0xA5, dtype=torch.uint8, device="cuda")
    d_off = torch.from_numpy(np.ascontiguousarray(off + base)).cuda()
    d_col = torch.from_numpy(np.ascontiguousarray(col + base)).cuda()
    s = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    assert L.b200spmv_csr_flat_analyze(s, C.c_int64(rows), C.c_int64(nnz), C.c_void_p(d_off.data_ptr()), C.c_int32(base),
                                       C.c_void_p(ws.data_ptr())) == 0
    h = C.c_int32(-1)
    assert L.b200spmv_csr_flat_hot_analyze(s, C.c_int(dtype), C.c_int64(rows), C.c_int64(cols), C.c_int64(nnz),
                                           C.c_void_p(d_col.data_ptr()), C.c_int32(base), C.c_void_p(ws.data_ptr()), C.byref(h)) == 0
    torch.cuda.synchronize()
    return ws, h.value, d_off, d_col


def _plan_case(case):
    if case == "rmat":
        off, col, _ = O.rmat_csr(200000, avg_nnz=16, seed=5, val_seed=6)
        return off, col, off.size - 1
    if case == "stencil":
        off, col, _ = O.gen_stencil5(300)
        return off, col, off.size - 1
    if case == "zipf":
        off, col = skewed_cols(30000, 60000, 12, 3)
        return off, col, 60000
    if case == "one_col":
        lens, cols = E.boundary_profiles(E.kernel_params())["one_col"]
    else:
        lens, cols = E.boundary_profiles(E.kernel_params())["rect_tall"]
    off, col = E.lens_to_structure(lens, cols, 0)
    return off, col, cols


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["rmat", "stencil", "zipf", "one_col", "rect_tall"])
@pytest.mark.parametrize("base", [0, 1])
@pytest.mark.parametrize("dtype", [0, 1])
def test_hot_plan_is_bit_exact(case, base, dtype):
    """The device hot plan (H, tau, the hot list and colp including its zero padding) against hot_plan() -- integer work, bit
    for bit -- in a workspace pre-filled with garbage."""
    import torch
    L = _lib()
    hb, mp, nb = _params(L)
    off, col, cols = _plan_case(case)
    ws, h, _, _ = _analyze(L, torch, off, col, base, cols, dtype)
    hot, tau, colp = hot_plan(col, 0, cols, hb, 8 if dtype else 4, mp, nb)
    oc, oh, ol = C.c_size_t(), C.c_size_t(), C.c_size_t()
    L.b200spmv_csr_flat_hot_offsets(C.c_int64(off.size - 1), C.c_int64(col.size), C.byref(oc), C.byref(oh))
    L.b200spmv_csr_flat_plan_offsets(C.c_int64(off.size - 1), C.c_int64(col.size), None, None, None, C.byref(ol))
    ctl = ws[ol.value:ol.value + 24].view(torch.int32).cpu().numpy()
    assert h == hot.size and (int(ctl[4]), int(ctl[5])) == (hot.size, tau)
    if case in ("rmat", "zipf", "one_col", "rect_tall"):
        assert h > 0, "these column laws are skewed enough for a hot plan"
    if case == "stencil":
        assert h == 0
    if h:
        assert np.array_equal(ws[oh.value:oh.value + 4 * h].view(torch.int32).cpu().numpy(), hot)
        assert np.array_equal(ws[oc.value:oc.value + 4 * colp.size].view(torch.int32).cpu().numpy(), colp)


def _mv(L, torch, ws, h, off_d, col_d, val, x, y0, base, alpha, beta, cols):
    y = y0.clone()
    dt = 1 if val.dtype == torch.float64 else 0
    npt = np.float64 if dt else np.float32
    a, b = np.array([alpha], npt), np.array([beta], npt)
    rc = L.b200spmv_csr_flat_mv(C.c_void_p(torch.cuda.current_stream().cuda_stream), C.c_int(dt), C.c_int64(off_d.numel() - 1),
                                C.c_int64(cols), C.c_int64(col_d.numel()), C.c_void_p(off_d.data_ptr()), C.c_void_p(col_d.data_ptr()),
                                C.c_void_p(val.data_ptr()), C.c_int32(base), C.c_void_p(a.ctypes.data), C.c_void_p(b.ctypes.data),
                                C.c_int(0), C.c_void_p(x.data_ptr()), C.c_void_p(y.data_ptr()), C.c_void_p(ws.data_ptr()), C.c_int32(h))
    assert rc == 0
    torch.cuda.synchronize()
    return y


EXACT_PROFILES = ["lane_ends", "chunk_and_cta_borders", "rows_cross_borders", "leading_trailing_empty", "one_col", "rect_tall",
                  "rect_wide", "random_mix_0"]


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["rmat"] + EXACT_PROFILES)
@pytest.mark.parametrize("kind", ["f32", "f64"])
@pytest.mark.parametrize("base", [0, 1])
@pytest.mark.parametrize("beta", [0.0, 0.5])
def test_hot_mv_is_bit_identical(case, kind, base, beta):
    """b200spmv_csr_flat_mv with the hot plan and with H = 0 on the same plan: torch.equal.  On the exact-arithmetic profiles
    both also equal the integer reference."""
    import torch
    L = _lib()
    tdt = torch.float64 if kind == "f64" else torch.float32
    if case == "rmat":
        off, col, val = O.rmat_csr(120000, avg_nnz=16, seed=11, val_seed=12, dtype=np.float64 if kind == "f64" else np.float32)
        cols = off.size - 1
        x = O.uniform(13, cols, val.dtype)
        y0 = O.uniform(14, off.size - 1, val.dtype)
        want = None
    else:
        lens, cols = E.boundary_profiles(E.kernel_params())[case]
        fx = E.Fixture(case, lens, cols, kind, seed=21)
        off, col, val, x, y0 = fx.off, fx.col, fx.val, fx.xf(), fx.y0f()
        fx.check(-2.0, beta)
        want = fx.want(-2.0, beta)
    ws, h, d_off, d_col = _analyze(L, torch, off, col, base, cols, 1 if kind == "f64" else 0)
    if case in ("rmat", "one_col", "rect_tall"):
        assert h > 0
    d_val, d_x, d_y0 = (torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in (val, x, y0))
    y_hot = _mv(L, torch, ws, h, d_off, d_col, d_val, d_x, d_y0, base, -2.0, beta, cols)
    y_cold = _mv(L, torch, ws, 0, d_off, d_col, d_val, d_x, d_y0, base, -2.0, beta, cols)
    assert y_hot.dtype == tdt and torch.equal(y_hot, y_cold)
    if want is not None:
        assert np.array_equal(y_hot.cpu().numpy().astype(np.float64), want)


@pytest.mark.gpu
def test_hot_mv_rejects_a_hot_count_beyond_the_budget():
    """H is the caller's: more hot slots than the packed copy holds for this value type is an argument error, not a launch."""
    import torch
    L = _lib()
    hb, _, _ = _params(L)
    off, col, cols = _plan_case("zipf")
    ws, h, d_off, d_col = _analyze(L, torch, off, col, 0, cols, 0)
    val = torch.ones(col.size, dtype=torch.float64, device="cuda")
    x = torch.ones(cols, dtype=torch.float64, device="cuda")
    y = torch.zeros(off.size - 1, dtype=torch.float64, device="cuda")
    one = np.array([1.0])
    for bad in (hb // 8 + 1, -1):
        rc = L.b200spmv_csr_flat_mv(C.c_void_p(torch.cuda.current_stream().cuda_stream), C.c_int(1), C.c_int64(off.size - 1),
                                    C.c_int64(cols), C.c_int64(col.size), C.c_void_p(d_off.data_ptr()), C.c_void_p(d_col.data_ptr()),
                                    C.c_void_p(val.data_ptr()), C.c_int32(0), C.c_void_p(one.ctypes.data), C.c_void_p(one.ctypes.data),
                                    C.c_int(0), C.c_void_p(x.data_ptr()), C.c_void_p(y.data_ptr()), C.c_void_p(ws.data_ptr()), C.c_int32(bad))
        assert rc == -1


@pytest.mark.gpu
def test_shim_runs_the_headline_matrix_on_a_hot_plan():
    """cusparseSpMV_preprocess builds the hot plan for a matrix that runs on csr_flat_kernel; cusparseSpMV then gives the bits
    the H = 0 path gives (flat kernel without preprocess of the hot part is not reachable through the shim, so compare with the
    direct call)."""
    import torch
    from cudalibrarysamples_b200 import cusparse_api as cs
    L = _lib()
    off, col, val = O.rmat_csr(100000, avg_nnz=16, seed=31, val_seed=32)
    rows = off.size - 1
    x = torch.from_numpy(O.uniform(33, rows)).cuda()
    api = cs.Api("b200")
    d = dict(off=torch.from_numpy(off).cuda(), col=torch.from_numpy(col).cuda(), val=torch.from_numpy(val).cuda())
    op = cs.SpMVOperator(api, "csr", rows, rows, d, preprocess=True)
    y = torch.zeros(rows, dtype=torch.float64, device="cuda")
    op(x, y, 1.0, 0.0)
    torch.cuda.synchronize()
    assert "csr_flat_kernel" in api.last_csr_kernel()
    op.close()
    ws, h, d_off, d_col = _analyze(L, torch, off, col, 0, rows, 1)
    assert h > 0
    y_cold = _mv(L, torch, ws, 0, d_off, d_col, d["val"], x, torch.zeros_like(y), 0, 1.0, 0.0, rows)
    assert torch.equal(y, y_cold)
