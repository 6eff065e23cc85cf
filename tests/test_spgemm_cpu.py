"""CPU: the SpGEMM numeric phase with structure reuse (DESIGN.md 3.28) without a GPU: the numpy restatement against scipy and against
an entry-by-entry loop, the plan-size formula, the route table, the header's declarations, and the helper's call sequence."""
import ctypes as C
import functools
import os
import sys

import numpy as np
import pytest
import scipy.sparse as sp
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from cudalibrarysamples_b200 import build  # noqa: E402
from cudalibrarysamples_b200 import cusparse_api as cs  # noqa: E402
from cudalibrarysamples_b200 import lib as _lib  # noqa: E402
from cudalibrarysamples_b200.lib import load, signatures  # noqa: E402
from oracle import spgemm_ref as R  # noqa: E402

CSR, COO = 1, 2              # cusparseFormat_t
I32, I64 = cs.CUSPARSE_INDEX_32I, cs.CUSPARSE_INDEX_64I
F32, F64, F16, C64 = cs.CUDA_R_32F, cs.CUDA_R_64F, cs.CUDA_R_16F, cs.CUDA_C_64F
INT_MAX = 2**31 - 1


def random_csr(rows, cols, density, seed, dtype, integer=False, empty_rows=()):
    rng = np.random.default_rng(seed)
    M = sp.random(rows, cols, density=density, random_state=seed, format="csr")
    M.data = rng.integers(-3, 4, M.nnz).astype(dtype) if integer else rng.uniform(-2, 2, M.nnz).astype(dtype)
    for i in empty_rows:
        M.data[M.indptr[i]:M.indptr[i + 1]] = 0
    M.eliminate_zeros() if empty_rows else None
    return M.indptr.astype(np.int32), M.indices.astype(np.int32), M.data.astype(dtype)


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_restatement_is_the_integer_product(dtype):
    """Integer-valued inputs: every partial sum is exact, so any order gives scipy's A @ B."""
    a = random_csr(40, 30, 0.2, 1, dtype, integer=True)
    b = random_csr(30, 50, 0.2, 2, dtype, integer=True)
    c_off, c_col = R.structural_pattern(a[0], a[1], b[0], b[1], 40, 50)
    got = R.spgemm(*a, *b, c_off, c_col)
    D = (sp.csr_matrix((a[2].astype(np.float64), a[1], a[0]), shape=(40, 30)) @
         sp.csr_matrix((b[2].astype(np.float64), b[1], b[0]), shape=(30, 50))).toarray()
    rows = np.repeat(np.arange(40), np.diff(c_off))
    assert np.array_equal(got, D[rows, c_col].astype(dtype))
    c0 = np.arange(len(c_col)).astype(dtype) % 7
    assert np.array_equal(R.spgemm(*a, *b, c_off, c_col, c0, 2.0, -3.0), (2 * D[rows, c_col] - 3 * c0).astype(dtype))


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("beta", [0.0, 0.75])
def test_restatement_is_the_entry_loop_bit_for_bit(dtype, beta):
    """Random values, unsorted A and B rows, empty A and B rows: the vectorised fold equals the plain per-entry loop."""
    a_off, a_col, a_val = random_csr(25, 20, 0.3, 3, dtype, empty_rows=(0, 7))
    b_off, b_col, b_val = random_csr(20, 30, 0.3, 4, dtype, empty_rows=(2, 5))
    rng = np.random.default_rng(5)
    for off, col, val in ((a_off, a_col, a_val), (b_off, b_col, b_val)):        # unsorted columns within each row
        for i in range(len(off) - 1):
            p = rng.permutation(off[i + 1] - off[i]) + off[i]
            col[off[i]:off[i + 1]], val[off[i]:off[i + 1]] = col[p].copy(), val[p].copy()
    c_off, c_col = R.structural_pattern(a_off, a_col, b_off, b_col, 25, 30)
    c0 = rng.uniform(-1, 1, len(c_col)).astype(dtype)
    got = R.spgemm(a_off, a_col, a_val, b_off, b_col, b_val, c_off, c_col, c0, 1.5, beta)
    want = R.spgemm_loop(a_off, a_col, a_val, b_off, b_col, b_val, c_off, c_col, c0, 1.5, beta)
    assert got.dtype == dtype and got.tobytes() == want.tobytes()


def test_restatement_skips_products_outside_the_pattern():
    a = (np.array([0, 2], np.int32), np.array([0, 1], np.int32), np.array([1.0, 2.0]))
    b = (np.array([0, 1, 2], np.int32), np.array([0, 3], np.int32), np.array([5.0, 7.0]))
    assert R.spgemm(*a, *b, np.array([0, 1], np.int32), np.array([3], np.int32)).tolist() == [14.0]


def test_products_per_row_and_traffic():
    a_off, a_col, _ = R.stencil5(6)
    per = R.products_per_row(a_off, a_col, a_off)
    assert per.dtype == np.int64 and per.sum() == np.diff(a_off)[a_col].sum()
    assert R.traffic_bytes(1, 1, 1, 1, 1, 8) == 2 * 4 * 2 + 16 + 12 + 12


@pytest.fixture(scope="module")
def shim():
    if not os.path.exists(build.LIB_PATH):
        pytest.skip("libb200spmv.so not built")
    return load(build.LIB_PATH)


def params(shim):
    w, warps, edges = C.c_int32(), C.c_int32(), (C.c_int64 * 3)()
    shim.b200spgemm_params(C.byref(w), C.byref(warps), edges)
    return w.value, warps.value, list(edges)


def test_plan_size_formula(shim):
    w, warps, edges = params(shim)
    assert w == 256 and warps == 8 and edges == [1 << 14, 1 << 10, 1 << 6]
    r256 = lambda b: (b + 255) // 256 * 256          # noqa: E731
    for rows, nnz_c in ((0, 0), (1, 1), (1000, 13000), (3, 10**6), (2**31 - 2, 2**31 - 2)):
        want = 256 + 2 * r256(4 * rows) + r256(8 * (rows + nnz_c // w + 1))
        assert shim.b200spgemm_plan_size(rows, 7, 9, nnz_c) == want
    assert shim.b200spgemm_plan_size(-1, 0, 0, 0) == 0


def route(shim, opA=0, opB=0, alg=0, ct=F64, fmt=(CSR, CSR, CSR), vt=(F64, F64, F64), idx=(I32, I32, I32), base=(0, 0, 0),
          sizes=(100, 80, 90, 500, 400, 2000)):
    return shim.b200spgemm_route(opA, opB, alg, ct, *fmt, *vt, *idx, *base, *sizes)


@pytest.fixture
def spgemm_on(shim):
    assert shim.b200spmv_set_option(b"B200SPMV_SPGEMM", b"on") == 0
    yield shim
    assert shim.b200spmv_set_option(b"B200SPMV_SPGEMM", b"auto") == 0


def test_route_default_mode_forwards_everything(shim):
    """No class has been measured at parity: in the default mode every call, in scope or not, goes to the closed library, so the
    size query answers the closed size untouched."""
    assert shim.b200spmv_set_option(b"B200SPMV_SPGEMM", b"auto") == 0
    assert shim.b200spmv_set_option(b"B200SPMV_SPGEMM", b"sometimes") == -1
    for ct in (F32, F64):
        for sizes in ((4, 4, 4, 9, 8, 12), (4 << 20, 4 << 20, 4 << 20, 20 << 20, 20 << 20, 50 << 20), (1 << 18, 1 << 18, 1 << 18, 2 << 20,
                                                                                                        2 << 20, 60 << 20)):
            assert route(shim, ct=ct, vt=(ct,) * 3, sizes=sizes) == 0


def test_route_under_on(spgemm_on):
    shim = spgemm_on
    for ct in (F32, F64):
        for alg in (cs.CUSPARSE_SPGEMM_DEFAULT, cs.CUSPARSE_SPGEMM_CSR_ALG_DETERMINITIC, cs.CUSPARSE_SPGEMM_CSR_ALG_NONDETERMINITIC):
            for base in ((0, 0, 0), (1, 1, 1), (1, 0, 1)):
                assert route(shim, alg=alg, ct=ct, vt=(ct,) * 3, base=base) == 1
    # the forwarded classes of the scope: transposes, ALG1-3, non-CSR operands, 16-bit / complex / mixed types, a compute type
    # other than the values', 64-bit or mixed indices, a base other than 0 / 1
    forwarded = [dict(opA=1), dict(opB=1), dict(opA=2), dict(alg=cs.CUSPARSE_SPGEMM_ALG1), dict(alg=4), dict(alg=5),
                 dict(fmt=(COO, CSR, CSR)), dict(fmt=(CSR, 5, CSR)), dict(fmt=(CSR, CSR, COO)),
                 dict(ct=F16, vt=(F16,) * 3), dict(ct=C64, vt=(C64,) * 3), dict(ct=F32, vt=(F32, F32, F32), fmt=(CSR, CSR, CSR), idx=(I64, I32, I32)),
                 dict(vt=(F32, F64, F64)), dict(vt=(F64, F32, F64)), dict(vt=(F64, F64, F32)), dict(ct=F32), dict(ct=F64, vt=(F32,) * 3),
                 dict(idx=(I64, I64, I64)), dict(idx=(I32, I32, -1)), dict(idx=(I32, I64, I32)), dict(base=(2, 0, 0)), dict(base=(0, 0, -1))]
    for kw in forwarded:
        assert route(shim, **kw) == 0, kw
    # every size below 2^31 - 1
    for k in range(6):
        sizes = [100, 80, 90, 500, 400, 2000]
        sizes[k] = INT_MAX - 1
        assert route(shim, sizes=tuple(sizes)) == 1, k
        sizes[k] = INT_MAX
        assert route(shim, sizes=tuple(sizes)) == 0, k
        sizes[k] = -1
        assert route(shim, sizes=tuple(sizes)) == 0, k


def test_declarations_are_live(shim):
    sigs = signatures("b200spmv.h")
    for name in ("b200spgemm_plan_size", "b200spgemm_params", "b200spgemm_plan", "b200spgemm_compute", "b200spgemm_route"):
        assert name in sigs and getattr(shim, name).argtypes == sigs[name][1]
    assert sigs["b200spgemm_plan_size"] == (C.c_size_t, [C.c_int64] * 4)
    with pytest.raises(C.ArgumentError):
        shim.b200spgemm_plan_size(C.c_double(1.0), 0, 0, 0)
    # host-side argument checks, before any CUDA call
    one = C.c_double(1.0)
    assert shim.b200spgemm_compute(None, 2, 4, 4, None, None, None, 0, None, None, None, 0, None, None, None, 0, C.addressof(one),
                                   C.addressof(one), 0, None) == -1
    assert shim.b200spgemm_plan(None, 4, 4, 4, 4, 4, 4, None, None, 0, None, 0, None, None, 0, None, 0, None, None) == -1
    assert shim.b200spgemm_plan(None, 4, 4, 4, 4, 4, 4, None, None, 2, None, 0, None, None, 0, None, 1 << 20, None, None) == -1


# ---- the helper's call sequence, under recorders that stand in for the libraries (as test_cusparse_api_trace_cpu.py does) -------
class _Recorder:
    def __init__(self):
        self.calls = []
        self.next_object = 0x1000

    def call(self, lib, name, *args):
        self.calls.append((lib, name))
        for a in args:
            o = getattr(a, "_obj", None)
            if isinstance(o, C.c_void_p):
                self.next_object += 0x10
                o.value = self.next_object
            elif isinstance(o, C.c_size_t):
                o.value = 8
            elif isinstance(o, C.c_int64) and name == "cusparseSpMatGetSize":
                o.value = 6
        return 0


class _Lib:
    def __init__(self, rec, name):
        self._rec, self._name = rec, name

    def __getattr__(self, fn):
        if fn.startswith("__"):
            raise AttributeError(fn)
        return functools.partial(self._rec.call, self._name, fn)


@pytest.mark.parametrize("impl", ["b200", "cusparse"])
def test_helper_runs_the_samples_call_sequence(monkeypatch, impl):
    """spgemm_reuse_example.c:138-218: createDescr, workEstimation (query, call), nnz (query, call), GetSize, CsrSetPointers, copy (query,
    call), compute; workEstimation, nnz and GetSize always on the closed library, and recompute is one more compute."""
    rec = _Recorder()
    for k in ("real", "shim"):
        monkeypatch.setattr(_lib, k, lambda k=k: _Lib(rec, k))
    monkeypatch.setattr(torch.cuda, "current_stream", lambda: type("S", (), {"cuda_stream": 0x5157})())
    api = cs.Api(impl)
    lib = "shim" if impl == "b200" else "real"
    t = lambda a, dt=torch.int32: torch.tensor(a, dtype=dt)          # noqa: E731
    A = dict(rows=2, cols=2, off=t([0, 1, 2]), col=t([0, 1]), val=t([1.0, 2.0], torch.float32))
    B = dict(rows=2, cols=3, off=t([0, 2, 3]), col=t([0, 2, 1]), val=t([1.0, 2.0, 3.0], torch.float32))
    r = cs.SpGEMMReuse(api, A, B)
    r.recompute(A["val"] * 2, B["val"] * 2, 1.0, 0.0)
    r.close()
    work = [(l, n) for l, n in rec.calls if not n.startswith(("cusparseCreateCsr", "cusparseDestroySpMat", "cusparseSetStream"))]
    assert work == [("real", "cusparseCreate"), (lib, "cusparseSpGEMM_createDescr"),
                    ("real", "cusparseSpGEMMreuse_workEstimation"), ("real", "cusparseSpGEMMreuse_workEstimation"),
                    ("real", "cusparseSpGEMMreuse_nnz"), ("real", "cusparseSpGEMMreuse_nnz"), ("real", "cusparseSpMatGetSize"),
                    (lib, "cusparseCsrSetPointers"), (lib, "cusparseSpGEMMreuse_copy"), (lib, "cusparseSpGEMMreuse_copy"),
                    (lib, "cusparseSpGEMMreuse_compute"), (lib, "cusparseSpGEMM_destroyDescr"), ("real", "cusparseDestroy")]
    assert [n for _, n in rec.calls].count("cusparseCreateCsr") == 3 and [n for _, n in rec.calls].count("cusparseDestroySpMat") == 3
    assert r.sizes == (8, 8, 8, 8, 8) and r.nnz == 6
