"""GPU: every SpMV / SpMM kernel of the library on the exact fixtures of oracle/exact.py, compared BIT FOR BIT.

On these inputs (nonzero small integers, power-of-two alpha / beta, even y0; a "wide" fp64 variant whose row sums need more than
fp32 has) every partial sum is exact, so any correct kernel returns exactly the int64 reference whatever its summation order,
atomics or split of a row between warps, CTAs and tiles.  np.array_equal replaces the relative-norm tolerances of
test_parity_gpu.py: a dropped, duplicated or narrowed product, a wrong row written, beta applied twice, y read when beta == 0
-- none of them hides under rounding.  The closed library runs on the same buffers and must be bit-equal too (a check on the
fixtures).  Every call goes through the C ABI and must have been served by our kernels (forwarded == 0, native + 1).

Axes: kernel x value type (fp32, fp64, fp64 wide) x index base x (fresh allocations | col / val / row views one element into
their allocation: naturally aligned, not 16-byte aligned); inside every test the scalar cases (1, 0) on a NaN-filled y,
(-2, 1/2), (-2, 1), (1/2, -1), in host and device pointer mode.  The semantic tests at the end: NaN / Inf in x (and in row 0
of B for SpMM), NaN stored in Sliced-ELL padding slots, and a structure-only plan reused after the values changed."""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import exact as E

pytestmark = pytest.mark.gpu

TORCH = {np.float32: torch.float32, np.float64: torch.float64}
KINDS = ["f32", "f64", "wide"]


@pytest.fixture(scope="module")
def cs():
    from cudalibrarysamples_b200 import cusparse_api
    return cusparse_api


@pytest.fixture(scope="module")
def b200(cs):
    return cs.Api("b200")


@pytest.fixture(scope="module")
def closed(cs):
    return cs.Api("cusparse")


@pytest.fixture(scope="module")
def P(b200):
    return E.kernel_params(b200.lib)


@pytest.fixture(scope="module")
def profiles(P):
    from test_parity_gpu import EDGE
    d = dict(E.boundary_profiles(P))
    for k in ("single_huge_row", "huge_then_tiny", "many_rows_end_in_one_step", "exactly_long", "all_empty", "trailing_empty"):
        d[f"edge_{k}"] = (EDGE[k], 120000)
    return d


_FIX = {}


def fixture(profiles, name, kind):
    key = (name, kind)
    if key not in _FIX:
        lens, cols = profiles[name]
        _FIX[key] = E.Fixture(name, lens, cols, kind, seed=11)
    return _FIX[key]


def dev(a, shift=False):
    """device copy of a; shift: a view that starts one element into its allocation (natural alignment only)"""
    t = torch.as_tensor(np.ascontiguousarray(a))
    if not shift:
        return t.cuda()
    buf = torch.zeros(t.numel() + 1, dtype=t.dtype, device="cuda")
    buf[1:] = t.cuda()
    return buf[1:]


def dev_padded(a):
    """device copy of a with 16 zero bytes on both sides (the view stays 16-byte aligned).  For the closed library's Sliced-ELL
    kernel: under index base 1 it reads x[-1] for padding entries (column 0 = -1 + base) and multiplies it by the padding
    value, so a NaN there reaches y, and x at the start of a device allocation makes it fault."""
    t = torch.as_tensor(np.ascontiguousarray(a))
    g = 16 // t.element_size()
    buf = torch.zeros(t.numel() + 2 * g, dtype=t.dtype, device="cuda")
    buf[g:g + t.numel()] = t.cuda()
    return buf[g:g + t.numel()]


def y_init(y0, beta, dtype):
    if beta == 0:
        return torch.full((max(len(y0), 0),), float("nan"), dtype=dtype, device="cuda")
    return dev(y0.astype(np.float64)).to(dtype)


def scalar(v, dtype, device_mode):
    return torch.tensor([v], dtype=dtype, device="cuda") if device_mode else v


def sweep(cs, api, fmt, rows, cols, arrays, x, y0, base=0, preprocess=True, transpose=False, xy_dtype=None, modes=(False, True),
          buffer=True):
    """One operator, every scalar case of E.SCALARS in each pointer mode: {(device_mode, alpha, beta): y (numpy)}.  For our
    library: every call ran on our kernels."""
    before = api.stats() if api.impl == "b200" else None
    op = cs.SpMVOperator(api, fmt, rows, cols, arrays, base=base, preprocess=preprocess, xy_dtype=xy_dtype,
                         op=cs.CUSPARSE_OPERATION_TRANSPOSE if transpose else cs.CUSPARSE_OPERATION_NON_TRANSPOSE)
    if not buffer:
        op.buffer = None                                   # NULL externalBuffer: no room for a plan
    out, calls = {}, 0
    try:
        for device_mode in modes:
            api.cusparseSetPointerMode(op.handle, cs.CUSPARSE_POINTER_MODE_DEVICE if device_mode else cs.CUSPARSE_POINTER_MODE_HOST)
            for alpha, beta in E.SCALARS:
                y = y_init(y0, beta, op.dtype)
                op(x, y, scalar(alpha, op.dtype, device_mode), scalar(beta, op.dtype, device_mode))
                torch.cuda.synchronize()
                out[(device_mode, alpha, beta)] = y.cpu().numpy()
                calls += 1
        api.cusparseSetPointerMode(op.handle, cs.CUSPARSE_POINTER_MODE_HOST)
    finally:
        op.close()
    if before is not None:
        after = api.stats()
        assert after["forwarded"] == before["forwarded"], "a call was forwarded to the closed library"
        assert after["native"] == before["native"] + calls
    return out


def assert_exact(out, want_of, what):
    for (device_mode, alpha, beta), got in out.items():
        want = want_of(alpha, beta)
        if not np.array_equal(got.astype(np.float64), want):
            bad = np.flatnonzero(got.astype(np.float64) != want)
            raise AssertionError(f"{what} device_mode={device_mode} alpha={alpha} beta={beta}: {bad.size} of {want.size} entries "
                                 f"differ, first at {bad[:5].tolist()}: got {got[bad[:5]].tolist()} want {want[bad[:5]].tolist()}")


# ------------------------------------------------------------------------------------------ CSR, every kernel
CSR_KERNELS = ["tile", "pipe", "ws", "rowwise", "seg", "seg:1", "seg:1000000", "flat", "short", "auto", "auto_nopre"]


@pytest.fixture(params=CSR_KERNELS)
def csr_kernel(request, b200):
    """as in test_parity_gpu.py, plus the default routing with and without cusparseSpMV_preprocess"""
    name, _, dense = request.param.partition(":")
    forced = name not in ("auto", "auto_nopre")
    b200.set_option("B200SPMV_FLAT", "on" if name == "flat" else ("off" if forced else "auto"))
    b200.set_option("B200SPMV_SHORT", "on" if name == "short" else ("off" if forced else "auto"))
    b200.set_option("B200SPMV_CSR_KERNEL", name if forced and name not in ("flat", "short") else "auto")
    b200.set_option("B200SPMV_SEG_DENSE", dense or "24")
    yield request.param
    b200.set_option("B200SPMV_CSR_KERNEL", "auto")
    b200.set_option("B200SPMV_SEG_DENSE", "24")
    b200.set_option("B200SPMV_FLAT", "auto")
    b200.set_option("B200SPMV_SHORT", "auto")


CSR_PROFILES = ["lane_ends", "chunk_and_cta_borders", "long_row_edges", "tile_border_ends", "rows_cross_borders", "short_block_caps",
                "leading_trailing_empty", "nnz_zero", "one_row", "one_col", "rect_tall", "rect_wide", "random_mix_0", "random_mix_1",
                "edge_single_huge_row", "edge_huge_then_tiny", "edge_many_rows_end_in_one_step", "edge_exactly_long", "edge_all_empty",
                "edge_trailing_empty"]


def csr_arrays(f, base, shift):
    return dict(off=dev(f.off + base), col=dev(f.col + base, shift), val=dev(f.val, shift))


@pytest.mark.parametrize("shift", [False, True], ids=["fresh", "offset_by_one"])
@pytest.mark.parametrize("base", [0, 1])
@pytest.mark.parametrize("kind", KINDS)
def test_csr_kernels_exact(cs, b200, closed, profiles, csr_kernel, kind, base, shift):
    for name in CSR_PROFILES:
        f = fixture(profiles, name, kind)
        arrays = csr_arrays(f, base, shift)
        x = dev(f.xf())
        out = sweep(cs, b200, "csr", f.rows, f.cols, arrays, x, f.y0f(), base, preprocess=csr_kernel != "auto_nopre")
        assert_exact(out, f.want, (csr_kernel, name))
        if csr_kernel == "auto" and f.nnz:          # the closed library on the same buffers: a check on the fixture
            lib = sweep(cs, closed, "csr", f.rows, f.cols, arrays, x, f.y0f(), base, modes=(False,))
            assert_exact(lib, f.want, ("closed library", name))


@pytest.mark.parametrize("shift", [False, True], ids=["fresh", "offset_by_one"])
@pytest.mark.parametrize("base", [0, 1])
@pytest.mark.parametrize("kind", KINDS)
def test_csr_transpose_exact(cs, b200, closed, profiles, kind, base, shift):
    for name in CSR_PROFILES:
        f = fixture(profiles, name, kind)
        arrays = csr_arrays(f, base, shift)
        out = sweep(cs, b200, "csr", f.rows, f.cols, arrays, dev(f.xf(True)), f.y0f(True), base, transpose=True)
        assert_exact(out, lambda a, b: f.want(a, b, transpose=True), ("csr transpose", name))


# ------------------------------------------------------------------------------------------ COO
@pytest.mark.parametrize("coo_kernel", ["tile", "seg"])
@pytest.mark.parametrize("order", ["sorted", "permuted"])
@pytest.mark.parametrize("shift", [False, True], ids=["fresh", "offset_by_one"])
@pytest.mark.parametrize("base", [0, 1])
@pytest.mark.parametrize("kind", KINDS)
def test_coo_kernels_exact(cs, b200, closed, profiles, coo_kernel, order, kind, base, shift):
    b200.set_option("B200SPMV_COO_KERNEL", coo_kernel)
    try:
        for name in CSR_PROFILES:
            f = fixture(profiles, name, kind)
            row = np.repeat(np.arange(f.rows, dtype=np.int32), np.diff(f.off))
            p = np.random.default_rng(3).permutation(f.nnz) if order == "permuted" else np.arange(f.nnz)
            arrays = dict(row=dev(row[p] + base, shift), col=dev(f.col[p] + base, shift), val=dev(f.val[p], shift))
            out = sweep(cs, b200, "coo", f.rows, f.cols, arrays, dev(f.xf()), f.y0f(), base)
            assert_exact(out, f.want, (coo_kernel, order, name))
            # the closed library on the same buffers -- fresh allocations only: its COO kernel faults on index / value arrays that
            # are not 16-byte aligned (cudaErrorMisalignedAddress on an H100, CUDA 12.9), where ours take the scalar path
            if order == "sorted" and coo_kernel == "seg" and not shift and f.nnz:
                lib = sweep(cs, closed, "coo", f.rows, f.cols, arrays, dev(f.xf()), f.y0f(), base, modes=(False,))
                assert_exact(lib, f.want, ("closed library", name))
    finally:
        b200.set_option("B200SPMV_COO_KERNEL", "auto")


# ------------------------------------------------------------------------------------------ Sliced-ELL
SELL_PROFILES = ["lane_ends", "short_block_caps", "leading_trailing_empty", "nnz_zero", "one_row", "one_col", "rect_tall", "rect_wide"]
SELL_SLICES = ["1", "2", "7", "32", "32_generic", "33", "64"]


@pytest.fixture
def sell_generic(b200):
    yield lambda on: b200.set_option("B200SPMV_SELL_GENERIC", "1" if on else "0")
    b200.set_option("B200SPMV_SELL_GENERIC", "0")


def sell_case(f, S, base, pad_val=0.0):
    """the fixture in Sliced-ELL; the first slice made only of empty rows (if any) gets two columns of padding"""
    lens = np.diff(f.off)
    empty = [s for s in range((f.rows + S - 1) // S) if not lens[s * S:(s + 1) * S].any()]
    return E.to_sell(f.off, f.col, f.val, S, base, min_width={empty[0]: 2} if empty else None, pad_val=pad_val)


@pytest.mark.parametrize("slice_size", SELL_SLICES)
@pytest.mark.parametrize("base", [0, 1])
@pytest.mark.parametrize("kind", KINDS)
def test_sell_kernels_exact(cs, b200, closed, profiles, sell_generic, slice_size, kind, base):
    S = int(slice_size.split("_")[0])
    sell_generic(slice_size.endswith("generic"))
    for name in SELL_PROFILES:
        f = fixture(profiles, name, kind)
        so, sc, sv = sell_case(f, S, base)
        arrays = dict(off=dev(so), col=dev(sc), val=dev(sv), slice_size=S, nnz=f.nnz)
        out = sweep(cs, b200, "sell", f.rows, f.cols, arrays, dev(f.xf()), f.y0f(), base)
        assert_exact(out, f.want, ("sell", slice_size, name))
        if f.nnz and slice_size in ("2", "32"):
            lib = sweep(cs, closed, "sell", f.rows, f.cols, arrays, dev_padded(f.xf()), f.y0f(), base, modes=(False,))
            assert_exact(lib, f.want, ("closed library", name))


# ------------------------------------------------------------------------------------------ the generic CSR kernels
GENERIC_CASES = {  # name -> (offsets int64, columns int64, kind); 64-bit offsets with 32-bit columns: cusparseCreateCsr refuses them
    "idx64_64": (True, True, "f64"), "idx64_64_f32": (True, True, "f32"),
    "wide_idx64": (True, True, "wide"), "fp32A_fp64xy": (False, False, "mixed"), "fp32A_fp64xy_idx64": (True, True, "mixed"),
}


@pytest.mark.parametrize("transpose", [False, True])
@pytest.mark.parametrize("base", [0, 1])
@pytest.mark.parametrize("case", list(GENERIC_CASES))
def test_generic_csr_exact(cs, b200, profiles, case, base, transpose):
    off64, col64, kind = GENERIC_CASES[case]
    for name in CSR_PROFILES[:12]:
        f = fixture(profiles, name, kind)
        arrays = dict(off=dev((f.off + base).astype(np.int64 if off64 else np.int32)),
                      col=dev((f.col + base).astype(np.int64 if col64 else np.int32)), val=dev(f.val))
        out = sweep(cs, b200, "csr", f.rows, f.cols, arrays, dev(f.xf(transpose)), f.y0f(transpose), base, transpose=transpose,
                    xy_dtype=TORCH[E.NP_XY[kind]])
        assert_exact(out, lambda a, b: f.want(a, b, transpose=transpose), (case, name))


@pytest.mark.parametrize("kind", KINDS)
def test_generic_csr_null_buffer_exact(cs, b200, profiles, kind):
    """NULL externalBuffer (no room for a plan): csr_generic_kernel serves the ordinary 32-bit call"""
    for name in CSR_PROFILES:
        f = fixture(profiles, name, kind)
        out = sweep(cs, b200, "csr", f.rows, f.cols, csr_arrays(f, 0, False), dev(f.xf()), f.y0f(), 0, preprocess=False, buffer=False)
        assert_exact(out, f.want, ("NULL buffer", name))


# ------------------------------------------------------------------------------------------ SpMM
def spmm(cs, api, f, B, C0, alpha, beta, ob, oc, base=0, pad=0, device_mode=False, shift=False):
    """C = alpha A B + beta C0 through cusparseSpMM with leading dimensions `pad` entries larger than tight; B (cols x n) and
    C0 (rows x n) int64 2-D.  Returns C (rows x n, float64)."""
    rows, cols, n = f.rows, f.cols, B.shape[1]
    npdt = E.NP_XY[f.kind]
    dt = TORCH[npdt]

    def pack(M, order, ld):
        r, c = M.shape
        if order == cs.CUSPARSE_ORDER_ROW:
            buf = np.full((r, ld), 7, npdt); buf[:, :c] = M
        else:
            buf = np.full((c, ld), 7, npdt); buf[:, :r] = M.T
        return buf.reshape(-1)

    ldb = (n if ob == cs.CUSPARSE_ORDER_ROW else cols) + pad
    ldc = (n if oc == cs.CUSPARSE_ORDER_ROW else rows) + pad
    Bd = dev(pack(B, ob, ldb))
    Cd = dev(pack(C0, oc, ldc)) if beta != 0 else torch.full((ldc * (rows if oc == cs.CUSPARSE_ORDER_ROW else n),), float("nan"),
                                                              dtype=dt, device="cuda")
    arrays = csr_arrays(f, base, shift)
    h = api.cusparseCreate()
    if device_mode:
        api.cusparseSetPointerMode(h, cs.CUSPARSE_POINTER_MODE_DEVICE)
    a_, b_ = scalar(alpha, dt, device_mode), scalar(beta, dt, device_mode)
    matA = api.cusparseCreateCsr(rows, cols, f.nnz, arrays["off"], arrays["col"], arrays["val"], base)
    matB = api.cusparseCreateDnMat(cols, n, ldb, Bd, ob)
    matC = api.cusparseCreateDnMat(rows, n, ldc, Cd, oc)
    op = cs.CUSPARSE_OPERATION_NON_TRANSPOSE
    ct = cs.CUDA_R_64F if dt == torch.float64 else cs.CUDA_R_32F
    before = api.stats() if api.impl == "b200" else None
    size = api.cusparseSpMM_bufferSize(h, op, op, a_, matA, matB, b_, matC, ct)
    buf = torch.empty(max(size, 16), dtype=torch.uint8, device="cuda")
    api.cusparseSpMM_preprocess(h, op, op, a_, matA, matB, b_, matC, ct, cs.CUSPARSE_SPMM_ALG_DEFAULT, buf)
    api.cusparseSpMM(h, op, op, a_, matA, matB, b_, matC, ct, cs.CUSPARSE_SPMM_ALG_DEFAULT, buf)
    torch.cuda.synchronize()
    if before is not None:
        after = api.stats()
        assert after["native"] == before["native"] + 1 and after["forwarded"] == before["forwarded"]
    api.cusparseDestroySpMat(matA); api.cusparseDestroyDnMat(matB); api.cusparseDestroyDnMat(matC); api.cusparseDestroy(h)
    out = Cd.cpu().numpy().astype(np.float64)
    if oc == cs.CUSPARSE_ORDER_ROW:
        Cm = out.reshape(rows, ldc)
        assert np.all(Cm[:, n:] == 7) or beta == 0, "SpMM wrote outside C"
        return Cm[:, :n]
    Cm = out.reshape(n, ldc)
    assert np.all(Cm[:, rows:] == 7) or beta == 0, "SpMM wrote outside C"
    return Cm[:, :rows].T


SPMM_PROFILES = ["lane_ends", "rect_tall", "rect_wide"]


@pytest.mark.parametrize("order_b,order_c", [(1, 1), (2, 2), (2, 1), (1, 2)])
@pytest.mark.parametrize("kind", KINDS)
def test_spmm_exact(cs, b200, closed, profiles, kind, order_b, order_c):
    for name in SPMM_PROFILES:
        f = fixture(profiles, name, kind)
        for i, n in enumerate((1, 3, 4, 63, 64, 65, 129)):
            _, B, _ = E.values(kind, 0, f.cols * n, 0, 100 + n)
            B = B.reshape(f.cols, n)
            C0 = E.values(kind, 0, 0, f.rows * n, 200 + n)[2].reshape(f.rows, n)
            E.check_spmm_exact(f.off, f.col, f.a, B, C0, f.p)
            base, pad, shift = i % 2, (3 if i % 3 == 0 else 0), i % 2 == 1
            for device_mode in (False, True):
                for alpha, beta in E.SCALARS:
                    got = spmm(cs, b200, f, B, C0, alpha, beta, order_b, order_c, base, pad, device_mode, shift)
                    want = E.spmm_reference(f.off, f.col, f.a, B, C0, alpha, beta)
                    assert np.array_equal(got, want), (name, n, order_b, order_c, device_mode, alpha, beta)
            if order_b == order_c and f.nnz and not shift:         # closed library: 16-byte aligned buffers only (see the COO test)
                got = spmm(cs, closed, f, B, C0, -2.0, 0.5, order_b, order_c, base, pad)
                assert np.array_equal(got, E.spmm_reference(f.off, f.col, f.a, B, C0, -2.0, 0.5)), ("closed library", name, n)


# ------------------------------------------------------------------------------------------ short kernel + dot
@pytest.mark.parametrize("kind", ["f32", "f64"])
def test_short_mv_dot_exact(b200, profiles, kind):
    """b200spmv_csr_short_mv_dot: y = A x and the fp64 dot y . x, both exact"""
    L = b200.lib
    L.b200spmv_csr_short_dot_workspace_bytes.restype = C.c_size_t
    f = fixture(profiles, "short_block_caps", kind)
    x = np.resize(f.x, max(f.rows, f.cols))[:f.cols]
    w = E.values(kind, 0, f.rows, 0, 5)[1]
    d_off, d_col, d_val, d_x, d_w = dev(f.off), dev(f.col), dev(f.val), dev(x.astype(E.NP_XY[kind])), dev(w.astype(E.NP_XY[kind]))
    ct = C.c_double if kind != "f32" else C.c_float
    for alpha, beta in E.SCALARS[:2]:
        y = y_init(f.y0, beta, TORCH[E.NP_XY[kind]])
        out = torch.zeros(1, dtype=torch.float64, device="cuda")
        ws = torch.zeros(int(L.b200spmv_csr_short_dot_workspace_bytes()), dtype=torch.uint8, device="cuda")
        rc = L.b200spmv_csr_short_mv_dot(C.c_void_p(torch.cuda.current_stream().cuda_stream), C.c_int(0 if kind == "f32" else 1),
                                         C.c_int64(f.rows), C.c_int64(f.cols), C.c_int64(f.nnz), C.c_void_p(d_off.data_ptr()),
                                         C.c_void_p(d_col.data_ptr()), C.c_void_p(d_val.data_ptr()), C.c_int32(0), C.byref(ct(alpha)),
                                         C.byref(ct(beta)), C.c_int(0), C.c_void_p(d_x.data_ptr()), C.c_void_p(y.data_ptr()),
                                         C.c_void_p(d_w.data_ptr()), C.c_void_p(out.data_ptr()), C.c_void_p(ws.data_ptr()))
        assert rc == 0
        torch.cuda.synchronize()
        want = E.reference(f.off, f.col, f.a, x, f.y0, alpha, beta)
        assert np.array_equal(y.cpu().numpy().astype(np.float64), want)
        assert float(out.item()) == float(np.dot((2 * want).astype(np.int64), w) / 2)


# ------------------------------------------------------------------------------------------ semantics: non-finite input
def nonfinite_x(f, transpose=False):
    """x with NaN at entry 0 (the column masked lanes default to) and +Inf at one other stored column"""
    x = f.xf(transpose).astype(np.float64)
    n = x.size
    used = np.unique(np.arange(f.rows) if transpose else f.col)
    inf_at = int(used[used != 0][len(used[used != 0]) // 2]) if np.any(used != 0) else (1 if n > 1 else None)
    x[0] = np.nan
    if inf_at is not None and inf_at < n:
        x[inf_at] = np.inf
    return x


def nonfinite_want(f, x, alpha, beta, transpose=False):
    """float64 over stored entries only (scipy): NaN / Inf where a row stores those columns, the exact value elsewhere"""
    import scipy.sparse as sp
    A = sp.csr_matrix((f.a.astype(np.float64), f.col, f.off), shape=(f.rows, f.cols))
    Ax = (A.T if transpose else A) @ x
    y0 = f.y0f(transpose).astype(np.float64)
    return alpha * Ax + (beta * y0 if beta != 0 else 0.0)


def same_nonfinite(got, want, lib, what):
    got = got.astype(np.float64)
    for arr, who in ((want, "reference"), (lib, "closed library")):
        if arr is None:
            continue
        arr = arr.astype(np.float64)
        assert np.array_equal(np.isnan(got), np.isnan(arr)), (what, who, "NaN mask", np.flatnonzero(np.isnan(got) != np.isnan(arr))[:8])
        assert np.array_equal(np.isposinf(got), np.isposinf(arr)) and np.array_equal(np.isneginf(got), np.isneginf(arr)), (what, who)
    fin = np.isfinite(want)
    assert np.array_equal(got[fin], want[fin]), (what, "finite rows")


NONFINITE_PROFILES = ["lane_ends", "chunk_and_cta_borders", "short_block_caps", "rows_cross_borders", "leading_trailing_empty", "rect_tall"]


@pytest.mark.parametrize("kind", ["f32", "f64"])
def test_nonfinite_x_csr(cs, b200, closed, profiles, csr_kernel, kind):
    for name in NONFINITE_PROFILES:
        f = fixture(profiles, name, kind)
        x = nonfinite_x(f)
        arrays = csr_arrays(f, 0, False)
        xd = dev(x.astype(E.NP_XY[kind]))
        out = sweep(cs, b200, "csr", f.rows, f.cols, arrays, xd, f.y0f(), 0, preprocess=csr_kernel != "auto_nopre", modes=(False,))
        lib = sweep(cs, closed, "csr", f.rows, f.cols, arrays, xd, f.y0f(), 0, modes=(False,))
        for k, got in out.items():
            same_nonfinite(got, nonfinite_want(f, x, k[1], k[2]), lib[k], (csr_kernel, name, k))


@pytest.mark.parametrize("kind", ["f32", "f64"])
def test_nonfinite_x_other_kernels(cs, b200, closed, profiles, sell_generic, kind):
    """COO (tile, seg), CSR^T, Sliced-ELL (sell32, sell_row, sell_generic), the generic CSR kernel (NULL buffer)"""
    for name in NONFINITE_PROFILES:
        f = fixture(profiles, name, kind)
        x = nonfinite_x(f)
        xd = dev(x.astype(E.NP_XY[kind]))
        row = np.repeat(np.arange(f.rows, dtype=np.int32), np.diff(f.off))
        coo = dict(row=dev(row), col=dev(f.col), val=dev(f.val))
        lib = sweep(cs, closed, "coo", f.rows, f.cols, coo, xd, f.y0f(), 0, modes=(False,))
        for kern in ("tile", "seg"):
            b200.set_option("B200SPMV_COO_KERNEL", kern)
            try:
                out = sweep(cs, b200, "coo", f.rows, f.cols, coo, xd, f.y0f(), 0, modes=(False,))
            finally:
                b200.set_option("B200SPMV_COO_KERNEL", "auto")
            for k, got in out.items():
                same_nonfinite(got, nonfinite_want(f, x, k[1], k[2]), lib[k], ("coo", kern, name, k))
        out = sweep(cs, b200, "csr", f.rows, f.cols, csr_arrays(f, 0, False), xd, f.y0f(), 0, preprocess=False, buffer=False, modes=(False,))
        for k, got in out.items():
            same_nonfinite(got, nonfinite_want(f, x, k[1], k[2]), lib[k], ("csr generic", name, k))
        for S, gen in ((32, False), (32, True), (7, False)):
            sell_generic(gen)
            so, sc, sv = sell_case(f, S, 0)
            arrays = dict(off=dev(so), col=dev(sc), val=dev(sv), slice_size=S, nnz=f.nnz)
            out = sweep(cs, b200, "sell", f.rows, f.cols, arrays, xd, f.y0f(), 0, modes=(False,))
            for k, got in out.items():
                same_nonfinite(got, nonfinite_want(f, x, k[1], k[2]), lib[k], ("sell", S, gen, name, k))
        xt = nonfinite_x(f, transpose=True)
        xtd = dev(xt.astype(E.NP_XY[kind]))
        out = sweep(cs, b200, "csr", f.rows, f.cols, csr_arrays(f, 0, False), xtd, f.y0f(True), 0, transpose=True, modes=(False,))
        libt = sweep(cs, closed, "csr", f.rows, f.cols, csr_arrays(f, 0, False), xtd, f.y0f(True), 0, transpose=True, modes=(False,))
        for k, got in out.items():
            same_nonfinite(got, nonfinite_want(f, xt, k[1], k[2], transpose=True), libt[k], ("csr transpose", name, k))


@pytest.mark.parametrize("order", [1, 2])
@pytest.mark.parametrize("kind", ["f32", "f64"])
def test_nonfinite_b_row0_spmm(cs, b200, closed, profiles, kind, order):
    """NaN / Inf in row 0 of B: only rows of C that store column 0 may turn non-finite -- as in the closed library"""
    import scipy.sparse as sp
    for name in ("lane_ends", "rect_tall", "leading_trailing_empty"):
        f = fixture(profiles, name, kind)
        for n in (1, 3, 5, 64, 65):
            _, B, _ = E.values(kind, 0, f.cols * n, 0, 300 + n)
            Bf = B.reshape(f.cols, n).astype(np.float64)
            Bf[0, :] = np.nan
            Bf[0, ::2] = np.inf
            A = sp.csr_matrix((f.a.astype(np.float64), f.col, f.off), shape=(f.rows, f.cols))
            want = -2.0 * (A @ Bf)
            got = spmm_float(cs, b200, f, Bf, -2.0, order)
            lib = spmm_float(cs, closed, f, Bf, -2.0, order)
            for j in range(n):
                same_nonfinite(got[:, j], want[:, j], lib[:, j], ("spmm", name, n, j))


def spmm_float(cs, api, f, Bf, alpha, order):
    """C = alpha A B (beta = 0, C NaN-filled) for a float64 B that may hold NaN / Inf"""
    dt = TORCH[E.NP_XY[f.kind]]
    rows, cols, n = f.rows, f.cols, Bf.shape[1]
    Bd = dev((Bf if order == 2 else Bf.T).astype(E.NP_XY[f.kind]).reshape(-1))
    Cd = torch.full((rows * n,), float("nan"), dtype=dt, device="cuda")
    arrays = csr_arrays(f, 0, False)
    Cb = cs.spmm(api, rows, cols, arrays, Bd, Cd, alpha, 0.0, order, order)
    out = Cb.cpu().numpy().astype(np.float64)
    return out.reshape(rows, n) if order == 2 else out.reshape(n, rows).T


# ------------------------------------------------------------------------------------------ semantics: Sliced-ELL padding values
@pytest.mark.parametrize("kind", ["f32", "f64"])
def test_sell_nan_in_padding_slots(cs, b200, closed, profiles, sell_generic, kind):
    """NaN stored in the VALUE of padding slots (column -1): what the closed library does with it, sell32 / sell_row /
    sell_generic must do too.  (The closed library skips padding entries: the result is the exact product.)"""
    for name in ("lane_ends", "leading_trailing_empty", "rect_tall"):
        f = fixture(profiles, name, kind)
        x = dev(f.xf())
        for S, gen in ((32, False), (32, True), (7, False), (7, True), (64, False)):
            so, sc, sv = sell_case(f, S, 0, pad_val=np.nan)
            assert np.isnan(sv).any()
            arrays = dict(off=dev(so), col=dev(sc), val=dev(sv), slice_size=S, nnz=f.nnz)
            lib = sweep(cs, closed, "sell", f.rows, f.cols, arrays, x, f.y0f(), 0, modes=(False,))
            nan_rows = {k: int(np.isnan(v).sum()) for k, v in lib.items()}
            print(f"closed library, NaN padding values, {name} S={S}: NaN rows per scalar case {nan_rows}")
            assert_exact(lib, f.want, ("closed library with NaN padding", name, S))
            sell_generic(gen)
            out = sweep(cs, b200, "sell", f.rows, f.cols, arrays, x, f.y0f(), 0)
            assert_exact(out, f.want, ("sell with NaN padding", name, S, gen))


# ------------------------------------------------------------------------------------------ semantics: the plan is structure only
@pytest.mark.parametrize("kernel", ["flat", "short", "seg", "tile", "auto"])
def test_plan_survives_new_values(cs, b200, profiles, kernel):
    """After cusparseSpMV_preprocess the plan depends on the structure only: overwrite val in place, call again -- the result
    is the exact product with the new values and no new analysis ran."""
    name = "short_block_caps" if kernel == "short" else "rows_cross_borders"
    f = fixture(profiles, name, "f64")
    b200.set_option("B200SPMV_FLAT", "on" if kernel == "flat" else ("auto" if kernel == "auto" else "off"))
    b200.set_option("B200SPMV_SHORT", "on" if kernel == "short" else ("auto" if kernel == "auto" else "off"))
    b200.set_option("B200SPMV_CSR_KERNEL", kernel if kernel in ("seg", "tile") else "auto")
    try:
        arrays = csr_arrays(f, 0, False)
        op = cs.SpMVOperator(b200, "csr", f.rows, f.cols, arrays, preprocess=True)
        a0 = b200.stats()["analyze"]
        x = dev(f.xf())
        for round_ in range(3):
            a = E.values("f64", f.nnz, 0, 0, 500 + round_)[0]
            arrays["val"].copy_(torch.as_tensor(a.astype(np.float64)))
            y = dev(f.y0f())
            op(x, y, -2.0, 0.5)
            torch.cuda.synchronize()
            want = E.reference(f.off, f.col, a, f.x, f.y0, -2.0, 0.5)
            assert np.array_equal(y.cpu().numpy(), want), (kernel, round_)
        assert b200.stats()["analyze"] == a0
        op.close()
    finally:
        b200.set_option("B200SPMV_CSR_KERNEL", "auto")
        b200.set_option("B200SPMV_FLAT", "auto")
        b200.set_option("B200SPMV_SHORT", "auto")
