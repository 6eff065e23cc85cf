"""GPU parity of spmv_generic.cu, CSR part -- the long tail of cusparseSpMV's real-valued argument space (SURVEY.md 8(f)-3):
64-bit indices (64/64 and 64/32), fp32 A with fp64 x / y / arithmetic, transposes of those, CSR calls without a workspace.
Every case goes through the C ABI (the cusparse* symbols of libb200spmv.so), is checked against the CPU oracle / scipy on
the same inputs and against the closed library on the same device buffers, and must be served by OUR kernels
(b200spmv_get_stats: forwarded unchanged).  A combination the closed library itself refuses must be refused by the shim
with the same status (cusparseSpMV_bufferSize keeps the real library's verdict).
The COO / Sliced-ELL kernels of the same file and the strided-batch SpMM are in tests/test_generic_opt_in_gpu.py.

Tolerances: fp64 arithmetic 1e-12, fp32 arithmetic 1e-5 (relative 2-norm), as in test_parity_gpu.py.
"""
import numpy as np
import pytest
import scipy.sparse as sp
import torch

from oracle import oracle as O

pytestmark = pytest.mark.gpu

NPI = {32: np.int32, 64: np.int64}
# (type of A's values, type of x / y / alpha / beta / the arithmetic)
TYPES = {"f64": (np.float64, torch.float64), "f32": (np.float32, torch.float32), "f32_f64": (np.float32, torch.float64)}
TOL = {torch.float64: 1e-12, torch.float32: 1e-5}


@pytest.fixture(scope="module")
def cs():
    from cudalibrarysamples_b200 import cusparse_api
    return cusparse_api


@pytest.fixture(scope="module")
def b200(cs):
    api = cs.Api("b200")
    api.set_option("B200SPMV_GENERIC", "csr")       # the library default
    return api


@pytest.fixture(scope="module")
def closed(cs):
    return cs.Api("cusparse")


def dev(a):
    return torch.as_tensor(a).cuda()


def relerr(got, want):
    got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
    n = np.linalg.norm(want)
    return np.linalg.norm(got - want) / (n if n > 0 else 1.0)


_CACHE = {}


def matrix(rows, cols, avg, seed):
    """Rectangular R-MAT (skewed rows, empty rows, a few very long rows), columns folded into [0, cols)."""
    key = (rows, cols, avg, seed)
    if key not in _CACHE:
        off, col, val = O.rmat_csr(rows, avg_nnz=avg, seed=seed, val_seed=seed + 1)
        _CACHE[key] = (off.astype(np.int64), (col % cols).astype(np.int64), val)
    return _CACHE[key]


def reference(off, col, val, rows, cols, x, y0, alpha, beta, transpose):
    A = sp.csr_matrix((val.astype(np.float64), col, off), shape=(rows, cols))
    Ax = (A.T if transpose else A) @ x.astype(np.float64)
    return alpha * Ax + (beta * y0.astype(np.float64) if beta != 0 else 0.0)


def spmv(cs, api, fmt, rows, cols, arrays, x, y, alpha, beta, base, transpose, xy_dtype, preprocess=True):
    """One cusparseSpMV through the C ABI; for our library the call must have run on our kernels."""
    before = api.stats() if api.impl == "b200" else None
    op = cs.SpMVOperator(api, fmt, rows, cols, arrays, base=base, preprocess=preprocess, xy_dtype=xy_dtype,
                         op=cs.CUSPARSE_OPERATION_TRANSPOSE if transpose else cs.CUSPARSE_OPERATION_NON_TRANSPOSE)
    op(x, y, alpha, beta)
    torch.cuda.synchronize()
    op.close()
    if before is not None:
        after = api.stats()
        assert after["forwarded"] == before["forwarded"], "the call was forwarded to the closed library"
        assert after["native"] == before["native"] + 1
    return y


def check(cs, b200, closed, fmt, rows, cols, arrays, host, base, transpose, types, alpha=-1.5, beta=0.5):
    """ours vs scipy / the oracle's arithmetic, ours vs the closed library; then beta = 0 on a NaN-filled y."""
    off, col, val = host
    _, xy = TYPES[types]
    nx, ny = (rows, cols) if transpose else (cols, rows)
    x = O.uniform(7, nx).astype(np.float64 if xy == torch.float64 else np.float32)
    y0 = O.uniform(8, ny).astype(x.dtype)
    want = reference(off, col, val, rows, cols, x, y0, alpha, beta, transpose)
    lib = closed_err = None
    try:
        lib = spmv(cs, closed, fmt, rows, cols, arrays, dev(x), dev(y0).clone(), alpha, beta, base, transpose, xy).cpu().numpy()
    except cs.CuSparseError as e:       # not a combination the closed library takes
        closed_err = e
    try:
        got = spmv(cs, b200, fmt, rows, cols, arrays, dev(x), dev(y0).clone(), alpha, beta, base, transpose, xy).cpu().numpy()
    except cs.CuSparseError as e:       # the shim may refuse only what the closed library refuses, with its status
        assert closed_err is not None and e.status == closed_err.status
        return
    assert relerr(got, want) < TOL[xy]
    if lib is not None:
        assert relerr(got, lib) < TOL[xy]
    y = torch.full((ny,), float("nan"), dtype=xy, device="cuda")
    got = spmv(cs, b200, fmt, rows, cols, arrays, dev(x), y, 1.0, 0.0, base, transpose, xy, preprocess=False).cpu().numpy()
    assert relerr(got, reference(off, col, val, rows, cols, x, y0, 1.0, 0.0, transpose)) < TOL[xy]


# ------------------------------------------------------------------------------------------ CSR
# (32-bit indices with one value type run on the specialised kernels: tests/test_parity_gpu.py)
CSR_CASES = [(o, c, t) for (o, c) in ((64, 64), (64, 32)) for t in ("f64", "f32", "f32_f64")] + [(32, 32, "f32_f64")]


@pytest.mark.parametrize("transpose", [False, True])
@pytest.mark.parametrize("off_bits,col_bits,types", CSR_CASES)
def test_csr_index_widths_and_mixed_precision(cs, b200, closed, off_bits, col_bits, types, transpose):
    rows, cols, base = 6000, 4100, 1
    off, col, val = matrix(rows, cols, 12, 201)
    va = val.astype(TYPES[types][0])
    arrays = dict(off=dev((off + base).astype(NPI[off_bits])), col=dev((col + base).astype(NPI[col_bits])), val=dev(va))
    check(cs, b200, closed, "csr", rows, cols, arrays, (off, col, va), base, transpose, types)


@pytest.mark.parametrize("avg", [2, 6, 40])
def test_csr_lane_counts_follow_the_mean_row_length(cs, b200, closed, avg):
    """4 / 8 / 32 lanes per row (launch_csr_generic picks them from nnz / rows; 16 lanes: the avg-12 cases above)."""
    rows = 5000
    off, col, val = matrix(rows, rows, avg, 300 + avg)
    arrays = dict(off=dev(off), col=dev(col), val=dev(val))
    check(cs, b200, closed, "csr", rows, rows, arrays, (off, col, val), 0, False, "f64", alpha=0.75, beta=-2.0)


def test_csr_edge_shapes_64bit(cs, b200, closed):
    """A single row holding everything; one column."""
    for off, col, rows, cols in (
        (np.array([0, 5000], np.int64), np.arange(5000, dtype=np.int64), 1, 5000),
        (np.arange(0, 1001, dtype=np.int64), np.zeros(1000, np.int64), 1000, 1),
    ):
        val = O.uniform(31, col.size)
        arrays = dict(off=dev(off), col=dev(col), val=dev(val))
        for transpose in (False, True):
            check(cs, b200, closed, "csr", rows, cols, arrays, (off, col, val), 0, transpose, "f64")


def test_csr_without_non_zeros_native_entry(cs):
    """rows x cols with no non-zero at all, through the native entry point (no descriptor, NULL index / value arrays):
    y = beta * y, and with beta = 0 y is overwritten without being read."""
    import ctypes as C
    from cudalibrarysamples_b200 import lib as L
    lib = L.shim()
    rows, cols = 300, 200
    off = dev(np.zeros(rows + 1, np.int64))
    stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    for transpose, ny in ((0, rows), (1, cols)):
        for beta, y in ((0.5, dev(O.uniform(9, ny))), (0.0, torch.full((ny,), float("nan"), dtype=torch.float64, device="cuda"))):
            want = beta * y.cpu().numpy() if beta else np.zeros(ny)
            a, b = C.c_double(2.0), C.c_double(beta)
            rc = lib.b200spmv_csr_generic_mv(stream, C.c_int(1), C.c_int(1), C.c_int(1), C.c_int(1), C.c_int(transpose), C.c_int64(rows),
                                             C.c_int64(cols), C.c_int64(0), C.c_void_p(off.data_ptr()), C.c_void_p(0), C.c_void_p(0),
                                             C.c_int64(0), C.byref(a), C.byref(b), C.c_int(0), C.c_void_p(0), C.c_void_p(y.data_ptr()))
            torch.cuda.synchronize()
            assert rc == 0
            assert np.array_equal(y.cpu().numpy(), want)


def test_csr_without_a_buffer_runs_on_the_generic_kernel(cs, b200):
    """A caller that passes externalBuffer = NULL (it ignored cusparseSpMV_bufferSize): no room for a plan, so the plan-free
    kernel serves the call -- rounds 1-2 forwarded it."""
    rows = 7000
    off, col, val = matrix(rows, rows, 12, 401)
    off32, col32 = off.astype(np.int32), col.astype(np.int32)
    x, y0 = O.uniform(1, rows), O.uniform(2, rows)
    h = b200.cusparseCreate()
    d_off, d_col, d_val, d_x, d_y = dev(off32), dev(col32), dev(val), dev(x), dev(y0)
    m = b200.cusparseCreateCsr(rows, rows, int(col.size), d_off, d_col, d_val)
    vx, vy = b200.cusparseCreateDnVec(rows, d_x), b200.cusparseCreateDnVec(rows, d_y)
    before = b200.stats()
    b200.cusparseSpMV(h, cs.CUSPARSE_OPERATION_NON_TRANSPOSE, 2.0, m, vx, -1.0, vy, cs.CUDA_R_64F, 0, None)
    torch.cuda.synchronize()
    after = b200.stats()
    assert after["native"] == before["native"] + 1 and after["forwarded"] == before["forwarded"]
    assert "csr_generic_kernel" in b200.last_csr_kernel()
    assert relerr(d_y.cpu().numpy(), O.spmv_csr(off32, col32, val, x, y0, 2.0, -1.0)) < 1e-12
    b200.cusparseDestroySpMat(m)
    b200.cusparseDestroyDnVec(vx)
    b200.cusparseDestroyDnVec(vy)
    b200.cusparseDestroy(h)


def test_generic_kernels_read_device_scalars(cs, b200):
    """CUSPARSE_POINTER_MODE_DEVICE (cusparse.h:275-278): alpha / beta are read inside the kernels."""
    rows, cols = 5000, 3000
    off, col, val = matrix(rows, cols, 12, 501)
    arrays = dict(off=dev(off), col=dev(col), val=dev(val))
    for transpose in (False, True):
        nx, ny = (rows, cols) if transpose else (cols, rows)
        x, y0 = O.uniform(3, nx), O.uniform(4, ny)
        op = cs.SpMVOperator(b200, "csr", rows, cols, arrays,
                             op=cs.CUSPARSE_OPERATION_TRANSPOSE if transpose else cs.CUSPARSE_OPERATION_NON_TRANSPOSE)
        b200.cusparseSetPointerMode(op.handle, cs.CUSPARSE_POINTER_MODE_DEVICE)
        y = dev(y0).clone()
        before = b200.stats()
        op(dev(x), y, dev(np.array([0.5])), dev(np.array([-3.0])))
        torch.cuda.synchronize()
        after = b200.stats()
        assert after["native"] == before["native"] + 1 and after["forwarded"] == before["forwarded"]
        b200.cusparseSetPointerMode(op.handle, cs.CUSPARSE_POINTER_MODE_HOST)
        op.close()
        assert relerr(y.cpu().numpy(), reference(off, col, val, rows, cols, x, y0, 0.5, -3.0, transpose)) < 1e-12
