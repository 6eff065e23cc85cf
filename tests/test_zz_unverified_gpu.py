"""GPU tests of the part of the library that is opt-in (B200SPMV_GENERIC=all) because it is not yet validated on the GPU:

  * coo_generic_kernel / sell_generic_kernel of spmv_generic.cu: COO and Sliced-ELL with 64-bit indices, fp32 A with fp64
    vectors, their transposes, Sliced-ELL transposes of any index width (SURVEY.md 8(f)-3);
  * strided-batch cusparseSpMM on our CSR x dense kernel (cuSPARSE/spmm_csr_batched/spmm_csr_batched_example.c:128-160).

Every test here is marked xfail(strict=False): `pytest -m gpu` reports them as XPASS or XFAIL
without turning the validated suite red, the file sorts last so that a fault here cannot disturb another test, and inside the
file the order is least risky first (the Sliced-ELL cases, where it is not known which index widths and transposes the
closed library itself accepts, come last).  The checks themselves are the usual ones: CPU oracle / scipy on the same inputs, the
closed library on the same device buffers (only with input it accepts), served by OUR kernels (forwarded unchanged).

Tolerances: fp64 arithmetic 1e-12, fp32 arithmetic 1e-5 (relative 2-norm), as in test_parity_gpu.py.
"""
import os
import subprocess

import numpy as np
import pytest
import scipy.sparse as sp
import torch

from oracle import oracle as O

pytestmark = [pytest.mark.gpu,
              pytest.mark.xfail(strict=False, reason="opt-in code path, not yet validated on the GPU")]
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

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
    api.set_option("B200SPMV_GENERIC", "all")       # opt in to the kernels under test
    yield api
    api.set_option("B200SPMV_GENERIC", "csr")       # back to the library default


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


# ------------------------------------------------------------------------------------------ strided-batch SpMM
def native(api, fn):
    before = api.stats()
    out = fn()
    after = api.stats()
    assert after["native"] == before["native"] + 1 and after["forwarded"] == before["forwarded"]
    return out


def test_batched_golden_exact(cs, b200):
    # spmm_csr_batched_example.c:56-88,183-196: fp32, column-major, shared row offsets, exact compare
    T = O.TOY_BATCHED
    C = native(b200, lambda: cs.spmm_batched(b200, 4, 4, 9, 2, dev(T["csr_off"]), dev(T["csr_col"].reshape(-1)), dev(T["val"].reshape(-1)),
                                             dev(T["B"].reshape(-1)), torch.zeros(24, device="cuda")))
    assert np.array_equal(C.cpu().numpy(), T["C"].reshape(-1))
    # the sample's "matA broadcast" alternative (:141-142): one matrix, two right-hand sides
    C = native(b200, lambda: cs.spmm_batched(b200, 4, 4, 9, 2, dev(T["csr_off"]), dev(T["csr_col"][0]), dev(T["val"][0]),
                                             dev(T["B"].reshape(-1)), torch.zeros(24, device="cuda"), colval_stride=0))
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


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
@pytest.mark.parametrize("order", [1, 2])
def test_batched_vs_oracle_and_cusparse(cs, b200, closed, dtype, order):
    """5 matrices with their own offsets / columns / values (offsets stride rows + 1), n = 40, alpha / beta != (1, 0)."""
    npdt = np.float32 if dtype == torch.float32 else np.float64
    rows, n, batches = 1500, 40, 5
    mats = [O.rmat_csr(rows, avg_nnz=9, seed=40 + i, val_seed=50 + i, dtype=npdt) for i in range(batches)]
    nnz = max(int(m[1].size) for m in mats)               # one nnz per batch entry: pad the shorter ones with explicit zeros in the last row
    offs, cols_, vals = [], [], []
    for off, col, val in mats:
        pad = nnz - col.size
        o = off.copy()
        o[-1] += pad
        offs.append(o)
        cols_.append(np.concatenate([col, np.zeros(pad, np.int32)]))
        vals.append(np.concatenate([val, np.zeros(pad, npdt)]))
    rng = np.random.default_rng(3)
    B = rng.uniform(-1, 1, (batches, rows, n)).astype(npdt)
    C0 = rng.uniform(-1, 1, (batches, rows, n)).astype(npdt)
    flat = (lambda M: M.reshape(-1)) if order == 2 else (lambda M: np.ascontiguousarray(M.transpose(0, 2, 1)).reshape(-1))
    args = (rows, rows, nnz, batches, dev(np.concatenate(offs)), dev(np.concatenate(cols_)), dev(np.concatenate(vals)), dev(flat(B)), dev(flat(C0)), -0.5, 2.0)
    got = native(b200, lambda: cs.spmm_batched(b200, *args, off_stride=rows + 1, order=order)).cpu().numpy()
    tol = 1e-5 if dtype == torch.float32 else 1e-12
    per = rows * n
    for i in range(batches):
        want = O.spmm_csr(offs[i], cols_[i], vals[i], B[i], C0[i], -0.5, 2.0, order_b="row", order_c="row")
        gi = got[per * i:per * (i + 1)].reshape((rows, n) if order == 2 else (n, rows))
        assert relerr(gi if order == 2 else gi.T, want) < tol, i
    try:
        lib = cs.spmm_batched(closed, *args, off_stride=rows + 1, order=order).cpu().numpy()
    except cs.CuSparseError:
        return                       # a batch layout the closed library does not take: the oracle comparison above stands
    assert relerr(got, lib) < tol


# ------------------------------------------------------------------------------------------ COO
@pytest.mark.parametrize("transpose", [False, True])
@pytest.mark.parametrize("types", ["f64", "f32", "f32_f64"])
def test_coo_64bit_indices_row_sorted(cs, b200, closed, types, transpose):
    """Row-sorted entries (what cusparseCreateCoo documents and spmv_coo_example.c:48-49 holds): ours vs scipy and vs the closed library."""
    rows, cols, base = 6000, 4100, 1
    off, col, val = matrix(rows, cols, 10, 601)
    va = val.astype(TYPES[types][0])
    row = np.repeat(np.arange(rows, dtype=np.int64), np.diff(off))
    arrays = dict(row=dev(row + base), col=dev(col + base), val=dev(va))
    check(cs, b200, closed, "coo", rows, cols, arrays, (off, col, va), base, transpose, types)


@pytest.mark.parametrize("transpose", [False, True])
def test_coo_64bit_indices_any_order(cs, b200, transpose):
    """Our COO kernels take the entries in any order (one RED.ADD per entry); the closed library is NOT run on this input."""
    rows, cols, base = 6000, 4100, 0
    off, col, val = matrix(rows, cols, 10, 601)
    row = np.repeat(np.arange(rows, dtype=np.int64), np.diff(off))
    perm = np.random.default_rng(5).permutation(col.size)
    arrays = dict(row=dev(row[perm]), col=dev(col[perm]), val=dev(val[perm]))
    nx, ny = (rows, cols) if transpose else (cols, rows)
    x, y0 = O.uniform(7, nx), O.uniform(8, ny)
    got = spmv(cs, b200, "coo", rows, cols, arrays, dev(x), dev(y0).clone(), -1.5, 0.5, base, transpose, torch.float64).cpu().numpy()
    assert relerr(got, reference(off, col, val, rows, cols, x, y0, -1.5, 0.5, transpose)) < 1e-12


# ------------------------------------------------------------------------------------------ Sliced-ELL
@pytest.mark.parametrize("types", ["f64", "f32", "f32_f64"])
@pytest.mark.parametrize("off_bits,col_bits,slice_size,transpose", [(64, 64, 32, False), (64, 32, 7, False), (64, 64, 7, True),
                                                                    (32, 32, 32, True), (32, 32, 7, True)])
def test_sell_index_widths_and_transposes(cs, b200, closed, off_bits, col_bits, slice_size, transpose, types):
    rows, cols, base = 5013, 3100, 0                                 # the last slice is partial
    off, col, val = matrix(rows, cols, 6, 701)
    va = val.astype(TYPES[types][0])
    so, sc, sv = O.csr_to_sell(off.astype(np.int32), col.astype(np.int32), va, slice_size)
    arrays = dict(off=dev(so.astype(NPI[off_bits])), col=dev(sc.astype(NPI[col_bits])), val=dev(sv), slice_size=slice_size,
                  nnz=int(col.size))
    check(cs, b200, closed, "sell", rows, cols, arrays, (off, col, va), base, transpose, types)


# ------------------------------------------------------------------------------------------ exact fixtures (oracle/exact.py)
@pytest.mark.parametrize("kind", ["f32", "f64", "wide", "mixed"])
@pytest.mark.parametrize("transpose", [False, True])
def test_coo_and_sell_generic_exact(cs, b200, kind, transpose):
    """coo_generic_kernel (64-bit indices) and sell_generic_kernel (A and A^T) on the exact fixtures: bit-equal to the int64
    reference, beta = 0 on a NaN-filled y included."""
    from oracle import exact as E
    lens = np.concatenate([[0, 3, 1, 0, 0, 40], np.full(70, 5), [600, 0, 1] * 5, [0, 0]])
    f = E.Fixture("mix", lens, 900, kind, seed=4)
    xy = torch.float64 if E.NP_XY[kind] == np.float64 else torch.float32
    row = np.repeat(np.arange(f.rows, dtype=np.int64), np.diff(f.off))
    coo = dict(row=dev(row), col=dev(f.col.astype(np.int64)), val=dev(f.val))
    so, sc, sv = E.to_sell(f.off, f.col, f.val, 7)
    sell = dict(off=dev(so.astype(np.int64)), col=dev(sc.astype(np.int64)), val=dev(sv), slice_size=7, nnz=f.nnz)
    for fmt, arrays in (("coo", coo), ("sell", sell)):
        for alpha, beta in E.SCALARS:
            y0 = f.y0f(transpose)
            y = torch.full((y0.size,), float("nan"), dtype=xy, device="cuda") if beta == 0 else dev(y0).to(xy)
            got = spmv(cs, b200, fmt, f.rows, f.cols, arrays, dev(f.xf(transpose)).to(xy), y, alpha, beta, 0, transpose, xy).cpu().numpy()
            assert np.array_equal(got.astype(np.float64), f.want(alpha, beta, transpose=transpose)), (fmt, alpha, beta)


@pytest.mark.parametrize("kind", ["f32", "f64"])
def test_batched_spmm_exact(cs, b200, kind):
    """strided-batch SpMM, three matrices sharing row offsets, on exact integer data: bit-equal to the int64 reference"""
    from oracle import exact as E
    rows, n, batches = 300, 33, 3
    f = E.Fixture("b", np.full(rows, 6), rows, kind, seed=6)
    npdt = E.NP_A[kind]
    vals = [E.values(kind, f.nnz, 0, 0, 40 + i)[0] for i in range(batches)]
    Bs = [E.values(kind, 0, rows * n, 0, 50 + i)[1].reshape(rows, n) for i in range(batches)]
    C0s = [E.values(kind, 0, 0, rows * n, 60 + i)[2].reshape(rows, n) for i in range(batches)]
    got = native(b200, lambda: cs.spmm_batched(b200, rows, rows, f.nnz, batches, dev(f.off), dev(np.tile(f.col, batches)),
                                               dev(np.concatenate(vals).astype(npdt)), dev(np.concatenate(Bs).astype(npdt).reshape(-1)),
                                               dev(np.concatenate(C0s).astype(npdt).reshape(-1)), -2.0, 0.5, order=2)).cpu().numpy()
    for i in range(batches):
        want = E.spmm_reference(f.off, f.col, vals[i], Bs[i], C0s[i], -2.0, 0.5)
        assert np.array_equal(got[rows * n * i:rows * n * (i + 1)].reshape(rows, n).astype(np.float64), want), i
