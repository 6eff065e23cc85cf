"""GPU: the opt-in routes of B200SPMV_GENERIC=all, checked strictly (no xfail):

  * coo_generic_kernel (COO with 64-bit indices, fp32 A with fp64 x / y / alpha / beta) through cusparseSpMV, A and A^T;
  * sell_generic_kernel<TRANSPOSE> (Sliced-ELL with 64-bit slice offsets or columns, every Sliced-ELL transpose, the mixed type);
  * the strided-batch loop of cusparseSpMM on a CSR A: one b200spmm_csr_ws call per matrix with A's offset and column / value
    strides, B's stride and C's stride.

Three kinds of check:
  * exact fixtures (oracle/exact.py): integer data on which every summation order gives the same bits, compared with the int64
    reference by np.array_equal, for every (alpha, beta) of E.SCALARS in host and device pointer mode, beta = 0 on a NaN-filled y;
  * R-MAT with uniform values against a long-double reference, componentwise:
        |y_i - yhat_i| <= gamma_{n_i + 2} * (|alpha| (|A| |x|)_i + |beta| |y0_i|),   gamma_k = k u / (1 - k u),
    n_i the stored entries of row i (column i for A^T), u the unit roundoff of the arithmetic type.  One row a few ulps off fails
    it.  The kernels add with atomics, so nothing here asserts bit-repeatability of those results;
  * routing: every call under test ran on our kernels (stats: native + 1, forwarded + 0), and under the default
    (B200SPMV_GENERIC=csr) the same calls are forwarded and give the closed library's bits.

The closed library is compared only where it accepts the call and, for Sliced-ELL, only at index base 0: under base 1 it reads
x[-1] for padding entries (see tests/test_exact_gpu.py).
"""
import os
import subprocess

import numpy as np
import pytest
import torch

from oracle import exact as E
from oracle import oracle as O

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

NPI = {32: np.int32, 64: np.int64}
TD = {np.float32: torch.float32, np.float64: torch.float64}
# random-value classes: (type of A's values, type of x / y / alpha / beta and of the arithmetic)
TYPES = {"f32": (np.float32, np.float32), "f64": (np.float64, np.float64), "f32_f64": (np.float32, np.float64)}
UNIT = {np.float32: 2.0 ** -24, np.float64: 2.0 ** -53}
KINDS = ["f32", "f64", "wide", "mixed"]           # exact fixtures; "mixed" is fp32 A with fp64 x / y (row sums past 2^24)
# (slice offsets, columns).  The closed library's cusparseCreateSlicedEll, which the shim forwards, refuses 64-bit offsets with
# 32-bit columns (CUSPARSE_STATUS_NOT_SUPPORTED, recorded by test_sell_closed_library_acceptance), so no SpMV can reach that pair.
SELL_WIDTHS = [(32, 32), (64, 64)]
SELL_WIDTHS_ALL = [(32, 32), (64, 32), (64, 64)]
SLICES = [1, 2, 7, 32, 33, 64]


@pytest.fixture(scope="module")
def cs():
    from cudalibrarysamples_b200 import cusparse_api
    return cusparse_api


@pytest.fixture(scope="module")
def b200(cs):
    api = cs.Api("b200")
    api.set_option("B200SPMV_GENERIC", "all")       # opt in to the kernels under test
    yield api
    api.set_option("B200SPMV_GENERIC", "csr")       # back to the library default


@pytest.fixture(scope="module")
def closed(cs):
    return cs.Api("cusparse")


class generic_option:
    """B200SPMV_GENERIC=value inside the block, "all" (the module's setting) after it"""

    def __init__(self, api, value):
        self.api, self.value = api, value

    def __enter__(self):
        self.api.set_option("B200SPMV_GENERIC", self.value)

    def __exit__(self, *exc):
        self.api.set_option("B200SPMV_GENERIC", "all")


def dev(a):
    return torch.as_tensor(np.ascontiguousarray(a)).cuda()


def status_of(cs, fn):
    """(0, result) or (cusparseStatus_t, None)"""
    try:
        return 0, fn()
    except cs.CuSparseError as e:
        return e.status, None


def counted(api, calls):
    """a context that asserts `calls` native calls and no forwarded one (our library), nothing for the closed one"""
    class _C:
        def __enter__(self):
            self.before = api.stats() if api.impl == "b200" else None

        def __exit__(self, exc_type, *rest):
            if exc_type is None and self.before is not None:
                after = api.stats()
                assert after["forwarded"] == self.before["forwarded"], "a call was forwarded to the closed library"
                assert after["native"] == self.before["native"] + calls, (after, self.before)
    return _C()


# ============================================================================================== SpMV: COO and Sliced-ELL
PROFILES = {   # name -> (row lengths, cols)
    "mix": ([0, 0, 3, 1, 0, 40] + [5] * 70 + [600, 0, 1] * 5 + [0, 0], 900),       # empty leading / trailing rows, long rows
    "huge_row": ([0, 0, 0, 3000, 0, 0, 0, 2], 3100),                               # one row holds nearly everything
    "nnz_zero": ([0] * 70, 50),
    "one_row": ([37], 64),
    "one_col": ([1] * 40 + [0, 1], 1),
}
_FIX, _SELL = {}, {}


def fixture(name, kind):
    if (name, kind) not in _FIX:
        lens, cols = PROFILES[name]
        _FIX[(name, kind)] = E.Fixture(name, lens, cols, kind, seed=21)
    return _FIX[(name, kind)]


def xy_torch(kind):
    return TD[E.NP_XY[kind]]


def sweep(cs, api, fmt, rows, cols, arrays, x, y0, base, transpose, xy_dtype):
    """One operator, every (alpha, beta) of E.SCALARS in host and device pointer mode: {(device, alpha, beta): y}.  Our library:
    every call native."""
    out = {}
    with counted(api, 2 * len(E.SCALARS)):
        op = cs.SpMVOperator(api, fmt, rows, cols, arrays, base=base, xy_dtype=xy_dtype,
                             op=cs.CUSPARSE_OPERATION_TRANSPOSE if transpose else cs.CUSPARSE_OPERATION_NON_TRANSPOSE)
        try:
            for device in (False, True):
                api.cusparseSetPointerMode(op.handle, cs.CUSPARSE_POINTER_MODE_DEVICE if device else cs.CUSPARSE_POINTER_MODE_HOST)
                for alpha, beta in E.SCALARS:
                    y = torch.full((max(y0.size, 1),), float("nan"), dtype=xy_dtype, device="cuda")
                    if beta != 0:
                        y[:y0.size] = dev(y0).to(xy_dtype)
                    sc = (lambda v: torch.tensor([v], dtype=xy_dtype, device="cuda")) if device else (lambda v: v)
                    op(dev(x).to(xy_dtype), y, sc(alpha), sc(beta))
                    torch.cuda.synchronize()
                    out[(device, alpha, beta)] = y[:y0.size].cpu().numpy()
        finally:
            op.close()
    return out


def assert_exact(out, f, transpose, what):
    for (device, alpha, beta), got in out.items():
        f.check(alpha, beta, transpose=transpose)
        assert np.array_equal(got.astype(np.float64), f.want(alpha, beta, transpose=transpose)), (what, device, alpha, beta)


def coo_arrays(f_off, f_col, val, idx, base, order, seed=5):
    row = np.repeat(np.arange(f_off.size - 1, dtype=np.int64), np.diff(f_off))
    col = np.asarray(f_col, np.int64)
    if order == "permuted":
        p = np.random.default_rng(seed).permutation(col.size)
        row, col, val = row[p], col[p], np.asarray(val)[p]
    return dict(row=dev((row + base).astype(NPI[idx])), col=dev((col + base).astype(NPI[idx])), val=dev(val))


@pytest.mark.parametrize("order", ["sorted", "permuted"])
@pytest.mark.parametrize("base", [0, 1])
@pytest.mark.parametrize("transpose", [False, True])
@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("idx", [32, 64])
def test_coo_exact(cs, b200, idx, kind, transpose, base, order):
    """COO through the shim on the exact fixtures: bit-equal to the int64 reference for every scalar case"""
    for name in PROFILES:
        f = fixture(name, kind)
        arrays = coo_arrays(f.off, f.col, f.val, idx, base, order)
        out = sweep(cs, b200, "coo", f.rows, f.cols, arrays, f.xf(transpose), f.y0f(transpose), base, transpose, xy_torch(kind))
        assert_exact(out, f, transpose, name)


def sell_of(f, S, base):
    """E.to_sell of the fixture with NaN in every padding slot, the first and the last slice widened past their longest row (on
    an all-empty slice: a slice of padding only)"""
    key = (f.name, f.kind, S, base)
    if key not in _SELL:
        ns = (f.rows + S - 1) // S
        lens = np.diff(f.off)
        w = [int(lens[s * S:(s + 1) * S].max()) for s in range(ns)]
        _SELL[key] = E.to_sell(f.off, f.col, f.val, S, base=base, min_width={0: w[0] + 2, ns - 1: w[-1] + 1}, pad_val=np.nan)
    return _SELL[key]


def sell_arrays(so, sc, sv, S, nnz, widths):
    return dict(off=dev(so.astype(NPI[widths[0]])), col=dev(sc.astype(NPI[widths[1]])), val=dev(sv), slice_size=S, nnz=nnz)


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("base", [0, 1])
@pytest.mark.parametrize("transpose", [False, True])
@pytest.mark.parametrize("widths", SELL_WIDTHS, ids=lambda w: f"{w[0]}_{w[1]}")
@pytest.mark.parametrize("S", SLICES)
def test_sell_exact(cs, b200, S, widths, transpose, base, kind):
    """Sliced-ELL through the shim on the exact fixtures (partial last slice, NaN padding, widened and padding-only slices):
    bit-equal to the int64 reference for every scalar case"""
    for name in PROFILES:
        f = fixture(name, kind)
        so, sc, sv = sell_of(f, S, base)
        assert np.isnan(sv).sum() == sv.size - f.nnz > 0
        arrays = sell_arrays(so, sc, sv, S, f.nnz, widths)
        out = sweep(cs, b200, "sell", f.rows, f.cols, arrays, f.xf(transpose), f.y0f(transpose), base, transpose, xy_torch(kind))
        assert_exact(out, f, transpose, name)


# ---------------------------------------------------------------------------------------------- random values, componentwise
_RMAT = {}


def rmat(rows, cols, avg, seed, a_type):
    key = (rows, cols, avg, seed, a_type)
    if key not in _RMAT:
        off, col, _ = O.rmat_csr(rows, cols, avg_nnz=avg, seed=seed, val_seed=seed + 1)
        val = np.random.default_rng(seed + 2).uniform(-1, 1, col.size).astype(a_type)
        _RMAT[key] = (off.astype(np.int64), col.astype(np.int64), val)
    return _RMAT[key]


def componentwise_bound(off, col, val, rows, cols, x, y0, alpha, beta, transpose, xy):
    """(yhat in long double, the bound gamma_{n_i + 2} (|alpha| (|A||x|)_i + |beta| |y0_i|)) for y = alpha op(A) x + beta y0"""
    row = np.repeat(np.arange(rows), np.diff(off))
    out_i, in_i, n_out = (col, row, cols) if transpose else (row, col, rows)
    ld = np.longdouble
    s = np.zeros(n_out, ld)
    np.add.at(s, out_i, val.astype(ld) * x.astype(ld)[in_i])
    mag = np.zeros(n_out, np.float64)
    np.add.at(mag, out_i, np.abs(val.astype(np.float64) * x.astype(np.float64)[in_i]))
    n = np.bincount(out_i, minlength=n_out).astype(np.float64) + 2
    u = UNIT[xy]
    gamma = n * u / (1 - n * u)
    yhat = ld(alpha) * s + ld(beta) * y0.astype(ld)
    bound = gamma * (abs(alpha) * mag + abs(beta) * np.abs(y0.astype(np.float64)))
    return yhat, bound * (1 + 2.0 ** -8)           # the slack covers the rounding of mag and of the long-double reference


def assert_componentwise(got, yhat, bound, what):
    err = np.abs(got.astype(np.longdouble) - yhat).astype(np.float64)
    bad = ~(err <= bound)
    assert not bad.any(), f"{what}: {bad.sum()} entries out of bound, first {np.flatnonzero(bad)[:5]}, " \
                          f"err {err[bad][:3]}, bound {bound[bad][:3]}"


def random_check(cs, b200, closed, fmt, rows, cols, arrays, host, base, transpose, types, compare_closed=True):
    off, col, val = host
    _, xy = TYPES[types]
    nx, ny = (rows, cols) if transpose else (cols, rows)
    x = np.random.default_rng(7).uniform(-1, 1, nx).astype(xy)
    y0 = np.random.default_rng(8).uniform(-1, 1, ny).astype(xy)
    alpha, beta = float(xy(-1.3)), float(xy(0.7))         # the scalars as the arithmetic type holds them
    op = cs.CUSPARSE_OPERATION_TRANSPOSE if transpose else cs.CUSPARSE_OPERATION_NON_TRANSPOSE

    def run(api):
        o = cs.SpMVOperator(api, fmt, rows, cols, arrays, base=base, xy_dtype=TD[xy], op=op)
        try:
            y = o(dev(x), dev(y0), alpha, beta)
            torch.cuda.synchronize()
            return y.cpu().numpy()
        finally:
            o.close()

    with counted(b200, 1):
        got = run(b200)
    yhat, bound = componentwise_bound(off, col, val, rows, cols, x, y0, alpha, beta, transpose, xy)
    assert_componentwise(got, yhat, bound, "ours")
    if compare_closed:
        st, lib = status_of(cs, lambda: run(closed))
        if st == 0:                                  # where the closed library takes the call, the two agree within both bounds
            assert np.all(np.abs(got.astype(np.float64) - lib.astype(np.float64)) <= 2 * bound)


@pytest.mark.parametrize("transpose", [False, True])
@pytest.mark.parametrize("types", list(TYPES))
@pytest.mark.parametrize("idx", [32, 64])
def test_coo_random_componentwise(cs, b200, closed, idx, types, transpose):
    """R-MAT (skewed rows, empty rows), row-sorted entries, base 1: within the componentwise bound, and next to the closed library"""
    rows, cols, base = 6000, 4100, 1
    off, col, val = rmat(rows, cols, 10, 601, TYPES[types][0])
    arrays = coo_arrays(off, col, val, idx, base, "sorted")
    random_check(cs, b200, closed, "coo", rows, cols, arrays, (off, col, val), base, transpose, types)


@pytest.mark.parametrize("transpose", [False, True])
@pytest.mark.parametrize("types", list(TYPES))
@pytest.mark.parametrize("idx", [32, 64])
def test_coo_random_any_order(cs, b200, idx, types, transpose):
    """the same with the entries in random order (our COO kernels take any order; the closed library is not run on it)"""
    rows, cols, base = 6000, 4100, 0
    off, col, val = rmat(rows, cols, 10, 601, TYPES[types][0])
    arrays = coo_arrays(off, col, val, idx, base, "permuted")
    random_check(cs, b200, None, "coo", rows, cols, arrays, (off, col, val), base, transpose, types, compare_closed=False)


@pytest.mark.parametrize("S", [7, 33])
@pytest.mark.parametrize("types", list(TYPES))
@pytest.mark.parametrize("transpose", [False, True])
@pytest.mark.parametrize("widths", SELL_WIDTHS, ids=lambda w: f"{w[0]}_{w[1]}")
def test_sell_random_componentwise(cs, b200, closed, widths, transpose, types, S):
    """R-MAT as Sliced-ELL (partial last slice), base 0: within the componentwise bound, and next to the closed library"""
    rows, cols = 5013, 3100
    off, col, val = rmat(rows, cols, 6, 701, TYPES[types][0])
    key = ("rmat", types, S)
    if key not in _SELL:
        _SELL[key] = E.to_sell(off, col, val, S)
    so, sc, sv = _SELL[key]
    arrays = sell_arrays(so, sc, sv, S, int(col.size), widths)
    random_check(cs, b200, closed, "sell", rows, cols, arrays, (off, col, val), 0, transpose, types)


# ---------------------------------------------------------------------------------------------- the default routing
def spmv_once(cs, api, fmt, f, arrays, transpose, kind):
    o = cs.SpMVOperator(api, fmt, f.rows, f.cols, arrays, xy_dtype=xy_torch(kind),
                        op=cs.CUSPARSE_OPERATION_TRANSPOSE if transpose else cs.CUSPARSE_OPERATION_NON_TRANSPOSE)
    try:
        y = o(dev(f.xf(transpose)), dev(f.y0f(transpose)), -2.0, 0.5)
        torch.cuda.synchronize()
        return y
    finally:
        o.close()


@pytest.mark.parametrize("kind", ["f64", "mixed"])
@pytest.mark.parametrize("transpose", [False, True])
@pytest.mark.parametrize("widths", SELL_WIDTHS_ALL, ids=lambda w: f"{w[0]}_{w[1]}")
def test_sell_closed_library_acceptance(cs, b200, closed, widths, transpose, kind):
    """Which Sliced-ELL index widths, transposes and types the closed library takes is recorded here (printed with -s), not
    assumed.  Under the default routing (B200SPMV_GENERIC=csr) the shim answers each call with the closed library's status and,
    when it accepts, its bits; only the 32-bit, single-type, non-transposed class runs natively there."""
    f = fixture("mix", kind)
    so, sc, sv = E.to_sell(f.off, f.col, f.val, 32)                 # base 0, zero padding
    arrays = sell_arrays(so, sc, sv, 32, f.nnz, widths)
    st_closed, lib = status_of(cs, lambda: spmv_once(cs, closed, "sell", f, arrays, transpose, kind))
    print(f"\n[closed library] Sliced-ELL offsets/columns {widths} transpose={transpose} {kind}: status {st_closed}")
    fast = widths == (32, 32) and not transpose and kind != "mixed"
    before = b200.stats()
    with generic_option(b200, "csr"):
        st, ours = status_of(cs, lambda: spmv_once(cs, b200, "sell", f, arrays, transpose, kind))
    after = b200.stats()
    assert st == st_closed
    if st == 0:
        assert after["native"] - before["native"] == (1 if fast else 0)
        assert after["forwarded"] - before["forwarded"] == (0 if fast else 1)
        assert torch.equal(ours, lib)
        assert np.array_equal(ours.cpu().numpy().astype(np.float64), f.want(-2.0, 0.5, transpose=transpose))


@pytest.mark.parametrize("case", ["coo_idx64_f64", "coo_idx64_f64_T", "coo_idx32_mixed", "coo_idx32_mixed_T"])
def test_coo_default_routing_forwards(cs, b200, closed, case):
    """Under B200SPMV_GENERIC=csr the COO classes of coo_generic_kernel are forwarded and give the closed library's bits"""
    idx, kind = (64, "f64") if "idx64" in case else (32, "mixed")
    transpose = case.endswith("_T")
    f = fixture("mix", kind)
    arrays = coo_arrays(f.off, f.col, f.val, idx, 0, "sorted")
    st_closed, lib = status_of(cs, lambda: spmv_once(cs, closed, "coo", f, arrays, transpose, kind))
    before = b200.stats()
    with generic_option(b200, "csr"):
        st, ours = status_of(cs, lambda: spmv_once(cs, b200, "coo", f, arrays, transpose, kind))
    after = b200.stats()
    assert st == st_closed
    assert after["native"] == before["native"]
    if st == 0:
        assert after["forwarded"] == before["forwarded"] + 1
        assert torch.equal(ours, lib)


# ============================================================================================== strided-batch CSR SpMM
SP_ROWS, SP_COLS = 37, 29                          # 37 rows: the column-major C kernel's 32-row tiles end inside the matrix
SP_LENS = [0, 3, 1, 0, 29, 2, 5, 0, 7] + [4] * 24 + [1, 0, 13, 0]
SP_NNZ = sum(SP_LENS)
# layout -> (per-matrix row offsets, per-matrix columns / values, per-matrix B)
LAYOUTS = {"strided": (True, True, True), "shared_off": (False, True, True), "broadcast_A": (False, False, True),
           "offsets_only": (True, False, True), "broadcast_B": (False, True, False)}
ORDERS = {"col_col": (1, 1), "col_row": (1, 2), "row_col": (2, 1), "row_row": (2, 2)}
CANARY = 7777.0


class BatchProblem:
    """An exact strided-batch product: matrix i is (offs[i], cols[i], vals[i]) (int64 values), B_i (cols x n) and C0_i
    (rows x n); the device arrays hold them in the layout's strides."""

    def __init__(self, kind, layout, batches, n, seed=0):
        self.kind, self.layout, self.batches, self.n = kind, layout, batches, n
        per_off, per_cv, per_b = LAYOUTS[layout]
        rng = np.random.default_rng(seed)
        rows, cols, nnz = SP_ROWS, SP_COLS, SP_NNZ
        self.offs, self.cols, self.vals = [], [], []
        for i in range(batches):
            lens = rng.permutation(SP_LENS) if per_off and i else np.asarray(SP_LENS)       # same nnz, other rows
            off, col = E.lens_to_structure(lens, cols, seed + 100 + (i if per_cv else 0))
            a = E.values(kind, nnz, 0, 0, seed + 200 + (i if per_cv else 0))[0]
            if not per_cv and i:                   # columns / values of matrix 0 under this matrix's row offsets
                col, a = self.cols[0], self.vals[0]
            self.offs.append(off)
            self.cols.append(col)
            self.vals.append(a)
        nb = batches if per_b else 1
        self.B = [E.values(kind, 0, cols * n, 0, seed + 300 + i)[1].reshape(cols, n) for i in range(nb)]
        self.C0 = [E.values(kind, 0, 0, rows * n, seed + 400 + i)[2].reshape(rows, n) for i in range(batches)]
        p = E.MANTISSA[kind]
        for i in range(batches):
            E.check_spmm_exact(self.offs[i], self.cols[i], self.vals[i], self.B[i if per_b else 0], self.C0[i], p)
        self.npdt = E.NP_A[kind]
        self.dtype = TD[self.npdt]
        self.off_stride = rows + 1 if per_off else 0
        self.colval_stride = nnz if per_cv else 0
        self.b_stride = None if per_b else 0       # broadcast B: B batched with stride 0 (the closed library refuses batch count 1)
        # device arrays; a shared col / val array gets (batches - 1) * (rows + 1) more valid entries behind it, so that reading it
        # at a row-offset stride stays inside the allocation (and gives wrong sums)
        self.d_off = dev(np.concatenate(self.offs) if per_off else self.offs[0])
        if per_cv:
            col_all, val_all = np.concatenate(self.cols), np.concatenate(self.vals)
        else:
            extra = (batches - 1) * (rows + 1)
            col_all = np.concatenate([self.cols[0], rng.integers(0, cols, extra)]).astype(np.int32)
            val_all = np.concatenate([self.vals[0], E.nonzero_ints(rng, extra, 1, 5)])
        self.d_col, self.d_val = dev(col_all.astype(np.int32)), dev(val_all.astype(self.npdt))

    def B_i(self, i):
        return self.B[i if len(self.B) > 1 else 0]

    def want(self, i, alpha, beta):
        return E.spmm_reference(self.offs[i], self.cols[i], self.vals[i], self.B_i(i), self.C0[i], alpha, beta)

    def dense_B(self, order_b):
        flat = [(b if order_b == 2 else b.T).reshape(-1) for b in self.B]
        return dev(np.concatenate(flat).astype(self.npdt))

    def c_layout(self, order_c, gap):
        """(ldc, elements of one C, batch stride): with a gap, ldc and the batch stride both exceed the tight ones"""
        rows, n = SP_ROWS, self.n
        ldc = (rows if order_c == 1 else n) + (3 if gap else 0)
        size = ldc * (n if order_c == 1 else rows)
        return ldc, size, size + (11 if gap else 0)

    def c_index(self, i, order_c, gap):
        """flat positions of C_i's rows x n entries in the C buffer"""
        ldc, _, stride = self.c_layout(order_c, gap)
        r, j = np.meshgrid(np.arange(SP_ROWS), np.arange(self.n), indexing="ij")
        return i * stride + (r + j * ldc if order_c == 1 else r * ldc + j)

    def dense_C(self, order_c, gap, beta):
        _, _, stride = self.c_layout(order_c, gap)
        buf = np.full(self.batches * stride, CANARY)
        for i in range(self.batches):
            buf[self.c_index(i, order_c, gap)] = self.C0[i] if beta != 0 else np.nan
        return dev(buf.astype(self.npdt))

    def check(self, C, order_c, gap, alpha, beta, what=""):
        got = C.cpu().numpy().astype(np.float64)
        live = np.zeros(got.size, bool)
        for i in range(self.batches):
            ix = self.c_index(i, order_c, gap)
            live[ix.reshape(-1)] = True
            assert np.array_equal(got[ix], self.want(i, alpha, beta)), (what, i, alpha, beta)
        assert np.all(got[~live] == CANARY), (what, "a gap between the matrices of C was written")


def run_batched(cs, api, P, order_b, order_c, gap, alpha, beta, buffer="auto", device_scalars=False):
    ldc, _, c_stride = P.c_layout(order_c, gap)
    sc = (lambda v: torch.tensor([v], dtype=P.dtype, device="cuda")) if device_scalars else (lambda v: v)
    with counted(api, 1):
        C = cs.spmm(api, SP_ROWS, SP_COLS, dict(off=P.d_off, col=P.d_col, val=P.d_val, nnz=SP_NNZ), P.dense_B(order_b),
                    P.dense_C(order_c, gap, beta), sc(alpha), sc(beta), order_b=order_b, order_c=order_c, n=P.n, ldc=ldc,
                    alg=cs.CUSPARSE_SPMM_CSR_ALG2, buffer=buffer, batches=P.batches, off_stride=P.off_stride,
                    colval_stride=P.colval_stride, b_stride=P.b_stride, b_batches=P.batches, compute=cs._VT[P.dtype],
                    preprocess=False, c_stride=c_stride)
        torch.cuda.synchronize()
    return C


_BP = {}


def batch_problem(kind, layout, batches, n):
    key = (kind, layout, batches, n)
    if key not in _BP:
        _BP[key] = BatchProblem(kind, layout, batches, n, seed=batches * 7 + n)
    return _BP[key]


@pytest.mark.parametrize("gap", [False, True], ids=["tight", "gap"])
@pytest.mark.parametrize("orders", list(ORDERS))
@pytest.mark.parametrize("n", [1, 63, 64, 65])
@pytest.mark.parametrize("batches", [1, 2, 5])
@pytest.mark.parametrize("layout", list(LAYOUTS))
@pytest.mark.parametrize("kind", ["f32", "f64"])
def test_batched_spmm_layouts_exact(cs, b200, kind, layout, batches, n, orders, gap):
    """Every batch layout, count, N and order pair, with and without an externalBuffer: C_i bit-equal to the int64 reference and
    the gaps of C (ldc past the tight one, batch stride past ldc * n) untouched.  With a column-major B, N >= 4 and a buffer,
    each product copies its own B_i row-major into the buffer first; every B_i differs, so a product that read an earlier copy
    fails here."""
    P = batch_problem(kind, layout, batches, n)
    ob, oc = ORDERS[orders]
    for buffer in ("auto", None):
        C = run_batched(cs, b200, P, ob, oc, gap, -2.0, 0.5, buffer=buffer)
        P.check(C, oc, gap, -2.0, 0.5, f"buffer={buffer}")
        C = run_batched(cs, b200, P, ob, oc, gap, 1.0, 0.0, buffer=buffer, device_scalars=True)
        P.check(C, oc, gap, 1.0, 0.0, f"buffer={buffer} device scalars")


@pytest.mark.parametrize("layout", list(LAYOUTS))
@pytest.mark.parametrize("kind", ["f32", "f64"])
def test_batched_spmm_exact(cs, b200, kind, layout):
    """Five products, N = 65, column-major B and C: every (alpha, beta) of E.SCALARS in host and device pointer mode, beta = 0 on
    a NaN-filled C, with and without an externalBuffer"""
    P = batch_problem(kind, layout, 5, 65)
    for buffer in ("auto", None):
        for device in (False, True):
            for alpha, beta in E.SCALARS:
                C = run_batched(cs, b200, P, 1, 1, True, alpha, beta, buffer=buffer, device_scalars=device)
                P.check(C, 1, True, alpha, beta, f"buffer={buffer} device={device}")


class Batched:
    """The batched SpMM call sequence on one handle, descriptors spelled out: batch counts of A, B and C set independently."""

    def __init__(self, cs, api, P, stream=None, a_batches=None, b_batches=None, b_stride=None, c_stride=None, order=1):
        self.api, self.P = api, P
        rows, cols, n = SP_ROWS, SP_COLS, P.n
        self.h = api.cusparseCreate()
        if stream is not None:
            api.cusparseSetStream(self.h, stream.cuda_stream)
        self.B = P.dense_B(order)
        self.C = P.dense_C(order, False, 0.0)
        self.A = api.cusparseCreateCsr(rows, cols, SP_NNZ, P.d_off, P.d_col, P.d_val, 0)
        self.matB = api.cusparseCreateDnMat(cols, n, cols if order == 1 else n, self.B, order)
        self.matC = api.cusparseCreateDnMat(rows, n, rows if order == 1 else n, self.C, order)
        self.ct = cs._VT[P.dtype]
        try:
            api.cusparseCsrSetStridedBatch(self.A, P.batches if a_batches is None else a_batches, P.off_stride, P.colval_stride)
            nb = (P.batches if len(P.B) > 1 else 1) if b_batches is None else b_batches
            if nb > 1:
                api.cusparseDnMatSetStridedBatch(self.matB, nb, cols * n if b_stride is None else b_stride)
            api.cusparseDnMatSetStridedBatch(self.matC, P.batches, rows * n if c_stride is None else c_stride)
            self.args = (self.h, cs.CUSPARSE_OPERATION_NON_TRANSPOSE, cs.CUSPARSE_OPERATION_NON_TRANSPOSE, 1.0, self.A, self.matB,
                         0.0, self.matC, self.ct, cs.CUSPARSE_SPMM_CSR_ALG2)
            size = api.cusparseSpMM_bufferSize(*self.args)
            self.buf = torch.empty(max(size, 16), dtype=torch.uint8, device="cuda")
        except Exception:
            self.close()
            raise

    def __call__(self):
        self.api.cusparseSpMM(*self.args, self.buf)

    def close(self):
        torch.cuda.synchronize()
        for d in (self.matC, self.matB):
            self.api.cusparseDestroyDnMat(d)
        self.api.cusparseDestroySpMat(self.A)
        self.api.cusparseDestroy(self.h)


def test_batched_on_a_side_stream(cs, b200):
    """The whole per-matrix launch sequence runs on the handle's stream: B is written on that stream behind a ~50 ms spin, so
    a launch on any other stream reads B before it is written"""
    P = batch_problem("f64", "strided", 5, 65)
    s = torch.cuda.Stream()
    q = Batched(cs, b200, P, stream=s)
    try:
        want_B = q.B.clone()
        q.B.zero_()
        torch.cuda.synchronize()
        with counted(b200, 1):
            with torch.cuda.stream(s):
                torch.cuda._sleep(100_000_000)
                q.B.copy_(want_B)
            q()
            s.synchronize()
        P.check(q.C, 1, False, 1.0, 0.0, "side stream")
    finally:
        q.close()


def test_batched_graph_replay(cs, b200):
    """The batched call captured in a CUDA graph on the handle's stream and replayed twice into a NaN-filled C"""
    P = batch_problem("f32", "strided", 5, 65)
    s = torch.cuda.Stream()
    q = Batched(cs, b200, P, stream=s)
    try:
        nan_c = q.C.clone()
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with counted(b200, 1):
            with torch.cuda.graph(g, stream=s):
                q()
        for rep in range(2):
            q.C.copy_(nan_c)
            torch.cuda.synchronize()
            g.replay()
            torch.cuda.synchronize()
            P.check(q.C, 1, False, 1.0, 0.0, f"replay {rep}")
        del g
    finally:
        q.close()


PARITY = {   # case -> (layout, Batched keyword arguments)
    "shared_offsets": ("shared_off", {}),
    "per_matrix_offsets": ("strided", {}),
    "B_batch_count_1": ("shared_off", dict(b_batches=1)),
    "B_stride_0": ("shared_off", dict(b_stride=0)),
    "A_batch_count_differs": ("shared_off", dict(a_batches=3)),
    "C_matrices_overlap": ("shared_off", dict(c_stride=SP_ROWS * 65 - 1)),
}


@pytest.mark.parametrize("case", list(PARITY))
def test_batched_status_parity(cs, b200, closed, case):
    """Batch layouts at and past the edge of what the closed library takes: our library answers with its status (printed with
    -s).  Where ours runs, C is bit-equal to the reference; where the closed library runs too, its C is compared with ours,
    except with per-matrix row offsets: there the closed library's C differs from the reference (whether it does is printed)."""
    layout, kw = PARITY[case]
    P = batch_problem("f64", layout, 5, 65)

    def run(api):
        q = Batched(cs, api, P, **kw)
        try:
            q()
            torch.cuda.synchronize()
            return q.C.clone()
        finally:
            q.close()

    st_closed, lib = status_of(cs, lambda: run(closed))
    st, ours = status_of(cs, lambda: run(b200))
    line = f"\n[closed library] batched CSR SpMM {case}: status {st_closed}; ours {st}"
    if st_closed == 0 and st == 0:
        line += f"; closed C equal to ours: {bool(torch.equal(ours, lib))}"
    print(line)
    assert st == st_closed
    if st == 0:
        got = ours.cpu().numpy().astype(np.float64)
        for i in range(P.batches):
            B = P.B[0] if case == "B_stride_0" else P.B[i]          # a stride-0 B: every product reads B_0
            want = E.spmm_reference(P.offs[i], P.cols[i], P.vals[i], B, P.C0[i], 1.0, 0.0)
            assert np.array_equal(got[P.c_index(i, 1, False)], want), (case, i)
        if layout == "shared_off":
            assert torch.equal(ours, lib)


def test_batched_default_routing_forwards(cs, b200, closed):
    """Under B200SPMV_GENERIC=csr a strided batch (shared row offsets, as in the sample) is forwarded and gives the closed
    library's bits"""
    P = batch_problem("f64", "shared_off", 5, 65)
    lib = run_batched(cs, closed, P, 1, 1, False, -2.0, 0.5)
    before = b200.stats()
    with generic_option(b200, "csr"):
        ours = cs.spmm(b200, SP_ROWS, SP_COLS, dict(off=P.d_off, col=P.d_col, val=P.d_val, nnz=SP_NNZ), P.dense_B(1),
                       P.dense_C(1, False, 0.5), -2.0, 0.5, n=P.n, alg=cs.CUSPARSE_SPMM_CSR_ALG2, batches=P.batches,
                       off_stride=P.off_stride, colval_stride=P.colval_stride, compute=cs._VT[P.dtype], preprocess=False)
        torch.cuda.synchronize()
    after = b200.stats()
    assert after["native"] == before["native"] and after["forwarded"] == before["forwarded"] + 1
    assert torch.equal(ours, lib)
    P.check(ours, 1, False, -2.0, 0.5, "forwarded")


def test_batched_golden_exact(cs, b200):
    """spmm_csr_batched_example.c's data (fp32, column-major, shared row offsets) and its "matA broadcast" variant, bit for bit"""
    T = O.TOY_BATCHED
    with counted(b200, 1):
        C = cs.spmm_batched(b200, 4, 4, 9, 2, dev(T["csr_off"]), dev(T["csr_col"].reshape(-1)), dev(T["val"].reshape(-1)),
                            dev(T["B"].reshape(-1)), torch.zeros(24, device="cuda"))
    assert np.array_equal(C.cpu().numpy(), T["C"].reshape(-1))
    with counted(b200, 1):
        C = cs.spmm_batched(b200, 4, 4, 9, 2, dev(T["csr_off"]), dev(T["csr_col"][0]), dev(T["val"][0]), dev(T["B"].reshape(-1)),
                            torch.zeros(24, device="cuda"), colval_stride=0)
    for i in range(2):
        want = O.spmm_csr(T["csr_off"], T["csr_col"][0], T["val"][0], T["B"][i].reshape(3, 4).T)
        assert np.array_equal(C.cpu().numpy()[12 * i:12 * i + 12], np.asfortranarray(want).T.reshape(-1))


def test_batched_sample_passes_through_the_shim():
    exe = os.path.join(ROOT, "oracle", "_ref", "spmm_csr_batched_example.b200")
    if not os.path.exists(exe):
        pytest.skip("oracle/_ref not built")
    env = {k: v for k, v in os.environ.items() if not k.startswith("B200SPMV_") and k != "LD_PRELOAD"}
    env["B200SPMV_LOG"] = "1"
    env["B200SPMV_GENERIC"] = "all"          # strided batches on our kernel are opt-in (csrc/config.h)
    p = subprocess.run([exe], capture_output=True, text=True, timeout=120, env=env)
    assert p.returncode == 0, p.stdout + p.stderr
    assert "spmm_csr_batched_example test PASSED" in p.stdout
    assert "[b200spmv] SpMM spmm_csr_kernel" in p.stderr and "batch=2" in p.stderr and "forwarded" not in p.stderr


@pytest.mark.parametrize("offsets", ["per_matrix", "shared"])
@pytest.mark.parametrize("orders", list(ORDERS))
@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
def test_batched_vs_oracle_and_cusparse(cs, b200, closed, dtype, orders, offsets):
    """Five R-MAT matrices with their own columns and values (and row offsets, or matrix 0's), N = 40, uniform values: every entry
    of every C_i within gamma_{n_i + 2} (|alpha| (|A_i| |B_i|) + |beta| |C0_i|) of a long-double reference.  With shared row
    offsets, the closed library's C within twice that of ours (it does not match the reference with per-matrix offsets, see
    test_batched_status_parity)."""
    npdt = np.float32 if dtype == torch.float32 else np.float64
    rows, n, batches = 1500, 40, 5
    ob, oc = ORDERS[orders]
    mats = [rmat(rows, rows, 9, 40 + i, npdt) for i in range(batches)]
    nnz = max(int(m[1].size) for m in mats)
    offs, cols_, vals = [], [], []
    for off, col, val in mats:                   # one nnz for the batch: the shorter matrices get more entries in the last row
        pad = nnz - col.size
        o = off.copy()
        o[-1] += pad
        offs.append(o)
        cols_.append(np.concatenate([col, np.arange(pad) % rows]))
        vals.append(np.concatenate([val, np.random.default_rng(9).uniform(-1, 1, pad).astype(npdt)]))
    if offsets == "shared":                      # matrix 0's row lengths, other sorted columns and values in every matrix
        for i in range(1, batches):
            offs[i] = offs[0]
            cols_[i] = E.lens_to_structure(np.diff(offs[0]), rows, 60 + i)[1]
            vals[i] = np.random.default_rng(70 + i).uniform(-1, 1, nnz).astype(npdt)
    rng = np.random.default_rng(3)
    B = rng.uniform(-1, 1, (batches, rows, n)).astype(npdt)
    C0 = rng.uniform(-1, 1, (batches, rows, n)).astype(npdt)
    flat = lambda M, order: (M if order == 2 else M.transpose(0, 2, 1)).reshape(-1)
    args = (rows, rows, dict(off=dev((np.concatenate(offs) if offsets == "per_matrix" else offs[0]).astype(np.int32)), col=dev(np.concatenate(cols_).astype(np.int32)),
                             val=dev(np.concatenate(vals)), nnz=nnz), dev(flat(B, ob)), dev(flat(C0, oc)), -0.5, 2.0)
    kw = dict(order_b=ob, order_c=oc, n=n, alg=cs.CUSPARSE_SPMM_CSR_ALG2, batches=batches,
              off_stride=rows + 1 if offsets == "per_matrix" else 0, colval_stride=nnz,
              compute=cs._VT[dtype], preprocess=False)
    with counted(b200, 1):
        got = cs.spmm(b200, *args, **kw).cpu().numpy()
        torch.cuda.synchronize()
    per = rows * n
    bounds = []
    for i in range(batches):
        gi = got[per * i:per * (i + 1)].reshape((rows, n) if oc == 2 else (n, rows))
        gi = gi if oc == 2 else gi.T
        b_i = []
        for j in range(n):                       # column j of C_i is an SpMV with x = B_i[:, j]
            yhat, bound = componentwise_bound(offs[i].astype(np.int64), cols_[i].astype(np.int64), vals[i], rows, rows, B[i][:, j],
                                              C0[i][:, j], -0.5, 2.0, False, npdt)
            assert_componentwise(gi[:, j], yhat, bound, f"C_{i} column {j}")
            b_i.append(bound)
        bounds.append(np.stack(b_i, 1))
    if offsets == "per_matrix":
        return
    st, lib = status_of(cs, lambda: cs.spmm(closed, *args, **kw).cpu().numpy())
    if st == 0:
        for i in range(batches):
            gi = got[per * i:per * (i + 1)].reshape((rows, n) if oc == 2 else (n, rows))
            li = lib[per * i:per * (i + 1)].reshape(gi.shape)
            bi = bounds[i] if oc == 2 else bounds[i].T
            assert np.all(np.abs(gi.astype(np.float64) - li.astype(np.float64)) <= 2 * bi)
