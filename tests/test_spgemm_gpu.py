"""GPU: cusparseSpGEMMreuse_compute on b200spgemm_compute (DESIGN.md 3.28) -- exact against scipy on small-integer inputs, bit for
bit against oracle/spgemm_ref.py on random values in every bin and on the long-row path, close to the closed library, reproducible
on a repeat and under CUDA-graph replay; the closed library's own behaviour pinned; the forwarded classes; the samples."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest
import scipy.sparse as sp
import torch

from oracle import spgemm_ref as R

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NP = {torch.float32: np.float32, torch.float64: np.float64}


@pytest.fixture(scope="module")
def cs():
    if not torch.cuda.is_available():
        pytest.skip("no GPU")
    from cudalibrarysamples_b200 import cusparse_api
    return cusparse_api


@pytest.fixture(scope="module")
def api(cs):
    return cs.Api("b200")


@pytest.fixture(scope="module")
def closed(cs):
    return cs.Api("cusparse")


@pytest.fixture
def on(api):
    api.set_option("B200SPMV_SPGEMM", "on")
    yield api
    api.set_option("B200SPMV_SPGEMM", "auto")


def dev(M, dtype, base=0):
    """CSR dict on the device from a scipy matrix (stored order kept)."""
    d = torch.device("cuda")
    return dict(rows=M.shape[0], cols=M.shape[1], off=torch.tensor(M.indptr + base, dtype=torch.int32, device=d),
                col=torch.tensor(M.indices + base, dtype=torch.int32, device=d), val=torch.tensor(M.data, dtype=dtype, device=d),
                base=base)


def csr(rows, cols, per_row_lengths, seed, values="int"):
    """rows x cols CSR with the given number of distinct columns per row (unsorted within a row), small integers or uniform values."""
    rng = np.random.default_rng(seed)
    off = np.concatenate([[0], np.cumsum(per_row_lengths)]).astype(np.int32)
    col = np.concatenate([rng.permutation(cols)[:n] for n in per_row_lengths] or [np.zeros(0, int)]).astype(np.int32)
    val = rng.integers(-3, 4, len(col)).astype(np.float64) if values == "int" else rng.uniform(-1, 1, len(col))
    return sp.csr_matrix((val, col, off), shape=(rows, cols))


def host(r):
    """(c_off, c_col) of a product, base 0, on the host."""
    off = r.c_off.cpu().numpy().astype(np.int64)
    base = int(off[0])
    return (off - base).astype(np.int32), (r.c_col[:r.nnz].cpu().numpy() - base).astype(np.int32)


def ref(A, B, c_off, c_col, dtype, c0=None, alpha=1.0, beta=0.0):
    nd = NP[dtype]
    return R.spgemm(A.indptr, A.indices, A.data.astype(nd), B.indptr, B.indices, B.data.astype(nd), c_off, c_col, c0, alpha, beta)


def native_count(api):
    return api.stats()["native"]


# ---------------------------------------------------------------------------------------------------- exact
@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
@pytest.mark.parametrize("bases", [(0, 0, 0), (1, 1, 1)])        # the closed workEstimation refuses mixed bases
@pytest.mark.parametrize("device_scalars", [False, True])
@pytest.mark.parametrize("beta", [0.0, 2.0])
def test_exact_small_integers(cs, on, dtype, bases, device_scalars, beta):
    A = csr(60, 50, np.random.default_rng(1).integers(0, 9, 60), 2)
    B = csr(50, 70, np.random.default_rng(3).integers(0, 9, 50), 4)
    r = cs.SpGEMMReuse(on, dev(A, dtype, bases[0]), dev(B, dtype, bases[1]), base_c=bases[2], device_alpha=device_scalars)
    c_off, c_col = host(r)
    rows = np.repeat(np.arange(60), np.diff(c_off))
    want = (A @ B).toarray()[rows, c_col]
    c0 = (np.arange(r.nnz) % 5).astype(NP[dtype])
    r.c_val[:r.nnz] = torch.tensor(c0, device="cuda")
    alpha, b = (torch.tensor([1.0], dtype=dtype, device="cuda"), torch.tensor([beta], dtype=dtype, device="cuda")) if device_scalars \
        else (1.0, beta)
    n0 = native_count(on)
    got = r.compute(alpha, b).cpu().numpy()
    assert native_count(on) == n0 + 1
    assert np.array_equal(got, (want + beta * c0).astype(NP[dtype]))
    r.close()


# ---------------------------------------------------------------------------------------------------- restatement
def bins_and_edges(L):
    w, warps, edges = C.c_int32(), C.c_int32(), (C.c_int64 * 3)()
    L.b200spgemm_params(C.byref(w), C.byref(warps), edges)
    return w.value, list(edges)


@pytest.fixture(scope="module")
def params(cs):
    from cudalibrarysamples_b200 import lib
    return bins_and_edges(lib.shim())


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
def test_restatement_every_bin_and_the_long_row(cs, on, params, dtype):
    """Random values, bit for bit against oracle/spgemm_ref.py: empty A rows, empty B rows, empty C rows, a C row longer than one
    window (three windows, each re-walking A's row), and rows whose product counts sit on every bin edge and one either side."""
    window, edges = params
    K, N = 16384, 16384
    rng = np.random.default_rng(7)
    b_len = rng.integers(0, 8, K)
    b_len[:64] = 0                                                        # empty B rows
    b_len[64] = 3 * window + 17                                           # one long B row: its A row gets a C row of > 3 windows
    B = csr(K, N, b_len, 8, values="uniform")
    a_rows = []
    a_rows.append([])                                                     # an empty A row
    a_rows.append([0, 1, 2])                                              # A row naming only empty B rows: an empty C row
    a_rows.append([64, 65, 66])                                           # the long row
    blen = np.diff(B.indptr)
    light = [k for k in range(65, K) if 1 <= blen[k] <= 7]
    for e in edges:                                                       # products edge - 1, edge, edge + 1
        for target in (e - 1, e, e + 1):
            row, tot = [], 0
            for k in rng.permutation(light):
                if tot + blen[k] <= target:
                    row.append(int(k)); tot += blen[k]
                if tot == target:
                    break
            assert tot == target
            a_rows.append(row)
    a_rows += [list(rng.choice(np.arange(65, K), rng.integers(1, 12), replace=False)) for _ in range(200)]
    lens = [len(r) for r in a_rows]
    A = sp.csr_matrix((rng.uniform(-1, 1, sum(lens)), np.concatenate([np.array(r, np.int32) for r in a_rows]),
                       np.concatenate([[0], np.cumsum(lens)])), shape=(len(a_rows), K))
    per = R.products_per_row(A.indptr, A.indices, B.indptr)
    for e in edges:
        assert {e - 1, e, e + 1} <= set(per.tolist())
    r = cs.SpGEMMReuse(on, dev(A, dtype), dev(B, dtype))
    c_off, c_col = host(r)
    assert np.diff(c_off)[1] == 0 and np.diff(c_off)[2] > 3 * window
    c0 = np.random.default_rng(9).uniform(-1, 1, r.nnz).astype(NP[dtype])
    for alpha, beta in ((1.0, 0.0), (-0.75, 1.25)):
        r.c_val[:r.nnz] = torch.tensor(c0, device="cuda")
        got = r.compute(alpha, beta).cpu().numpy()
        want = ref(A, B, c_off, c_col, dtype, c0, alpha, beta)
        assert got.tobytes() == want.tobytes(), np.flatnonzero(got != want)[:10]
    r.close()


# ---------------------------------------------------------------------------------------------------- against the closed library
@pytest.mark.parametrize("dtype,tol", [(torch.float32, 1e-5), (torch.float64, 1e-12)])
@pytest.mark.parametrize("shape", ["stencil", "rmat", "rectangular"])
def test_close_to_the_closed_library(cs, on, closed, dtype, tol, shape):
    if shape == "stencil":
        off, col, val = R.stencil5(64)
        A = B = sp.csr_matrix((val, col, off))
    elif shape == "rmat":
        off, col, val = R.rmat(12, 8, 3)
        A = B = sp.csr_matrix((val, col, off), shape=(1 << 12, 1 << 12))
    else:
        off, col, val = R.restriction2(64)
        A = sp.csr_matrix((val, col, off), shape=(32 * 32, 64 * 64))
        o2, c2, v2 = R.stencil5(64)
        B = sp.csr_matrix((v2, c2, o2))
    ours = cs.SpGEMMReuse(on, dev(A, dtype), dev(B, dtype))
    theirs = cs.SpGEMMReuse(closed, dev(A, dtype), dev(B, dtype))
    assert torch.equal(ours.c_off, theirs.c_off) and torch.equal(ours.c_col[:ours.nnz], theirs.c_col[:theirs.nnz])
    a = ours.compute(1.0, 0.0).double()
    b = theirs.compute(1.0, 0.0).double()
    assert (torch.linalg.norm(a - b) / torch.linalg.norm(b)).item() < tol
    ours.close(); theirs.close()


# ---------------------------------------------------------------------------------------------------- reuse
@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
def test_reuse_repeat_and_graph_replay(cs, on, dtype):
    off, col, val = R.rmat(11, 8, 5)
    A = sp.csr_matrix((val, col, off), shape=(1 << 11, 1 << 11))
    r = cs.SpGEMMReuse(on, dev(A, dtype), dev(A, dtype))
    c_off, c_col = host(r)
    r.compute()
    rng = np.random.default_rng(11)
    a2 = rng.uniform(-1, 1, A.nnz)
    b2 = rng.uniform(-1, 1, A.nnz)
    first = r.recompute(torch.tensor(a2, dtype=dtype, device="cuda"), torch.tensor(b2, dtype=dtype, device="cuda")).clone()
    A2, B2 = sp.csr_matrix((a2, col, off), shape=A.shape), sp.csr_matrix((b2, col, off), shape=A.shape)
    assert first.cpu().numpy().tobytes() == ref(A2, B2, c_off, c_col, dtype).tobytes()
    assert torch.equal(r.compute(), first)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    g = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s):
        on.cusparseSetStream(r.handle, s.cuda_stream)
        with torch.cuda.graph(g, stream=s):
            r.compute()
    torch.cuda.synchronize()
    r.c_val.fill_(float("nan"))
    for _ in range(3):
        g.replay()
    torch.cuda.synchronize()
    assert torch.equal(r.c_val[:r.nnz], first)
    on.cusparseSetStream(r.handle, torch.cuda.current_stream().cuda_stream)
    r.close()


# ---------------------------------------------------------------------------------------------------- the closed library, pinned
@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
def test_closed_behaviour_pinned_and_matched(cs, on, closed, dtype):
    """The closed reuse_copy leaves C's columns strictly ascending even for unsorted A and B rows and zeroes C's values; its
    compute applies beta != 0 as alpha AB + beta C and does not read C at beta = 0 (a NaN there stays out).  Ours does the same."""
    A = csr(80, 60, np.random.default_rng(1).integers(0, 10, 80), 12)
    B = csr(60, 90, np.random.default_rng(2).integers(0, 10, 60), 13)
    for a in (closed, on):
        r = cs.SpGEMMReuse(a, dev(A, dtype), dev(B, dtype))
        c_off, c_col = host(r)
        assert all(np.all(np.diff(c_col[c_off[i]:c_off[i + 1]]) > 0) for i in range(80))
        assert bool((r.c_val[:r.nnz] == 0).all())
        rows = np.repeat(np.arange(80), np.diff(c_off))
        want = (A @ B).toarray()[rows, c_col]
        c0 = (np.arange(r.nnz) % 5 + 1).astype(NP[dtype])
        r.c_val[:r.nnz] = torch.tensor(c0, device="cuda")
        assert np.array_equal(r.compute(3.0, 0.5).cpu().numpy(), (3 * want + 0.5 * c0).astype(NP[dtype]))
        r.c_val[:r.nnz] = float("nan")
        assert np.array_equal(r.compute(1.0, 0.0).cpu().numpy(), want.astype(NP[dtype]))
        r.close()


# ---------------------------------------------------------------------------------------------------- forwarding
def test_default_mode_forwards_with_the_closed_size_and_result(cs, api, closed):
    A = csr(50, 40, np.random.default_rng(4).integers(0, 6, 50), 14, values="uniform")
    api.set_option("B200SPMV_SPGEMM", "auto")
    n0, f0 = api.stats()["native"], api.stats()["forwarded"]
    ours = cs.SpGEMMReuse(api, dev(A.T.tocsr(), torch.float64), dev(A, torch.float64))
    theirs = cs.SpGEMMReuse(closed, dev(A.T.tocsr(), torch.float64), dev(A, torch.float64))
    assert ours.sizes == theirs.sizes
    assert torch.equal(ours.compute(), theirs.compute())
    st = api.stats()
    assert st["native"] == n0 and st["forwarded"] == f0 + 1
    ours.close(); theirs.close()


def test_size_query_adds_the_plan_under_on(cs, on, closed):
    A = csr(50, 40, np.random.default_rng(4).integers(0, 6, 50), 14, values="uniform")
    ours = cs.SpGEMMReuse(on, dev(A.T.tocsr(), torch.float32), dev(A, torch.float32))
    theirs = cs.SpGEMMReuse(closed, dev(A.T.tocsr(), torch.float32), dev(A, torch.float32))
    plan = on.lib.b200spgemm_plan_size(40, int(A.nnz), int(A.nnz), ours.nnz)
    assert ours.sizes[:4] == theirs.sizes[:4] and ours.sizes[4] == (theirs.sizes[4] + 255) // 256 * 256 + plan
    ours.close(); theirs.close()


@pytest.mark.parametrize("case", ["alg1", "compute_type", "small_buffer", "new_a_pattern_pointer"])
def test_forwarded_cases_give_the_closed_result(cs, on, closed, case):
    A = csr(70, 70, np.random.default_rng(5).integers(0, 7, 70), 15, values="uniform")
    kw = dict(alg=cs.CUSPARSE_SPGEMM_ALG1) if case == "alg1" else {}
    if case == "small_buffer":                                           # the closed size only: no room for a plan
        probe = cs.SpGEMMReuse(closed, dev(A, torch.float64), dev(A, torch.float64))
        kw = dict(buffer5=probe.sizes[4])
        probe.close()
    try:
        theirs = cs.SpGEMMReuse(closed, dev(A, torch.float64), dev(A, torch.float64), **{k: v for k, v in kw.items() if k == "alg"})
    except cs.CuSparseError as e:
        pytest.skip(f"the closed library refuses the reuse set-up of this class: {e}")
    ours = cs.SpGEMMReuse(on, dev(A, torch.float64), dev(A, torch.float64), **kw)
    if case == "compute_type":
        ours.compute_type = theirs.compute_type = cs.CUDA_R_32F
    if case == "new_a_pattern_pointer":                                  # same pattern, new arrays: the plan no longer applies
        d = dev(A, torch.float64)
        ours._keep = d
        on.cusparseCsrSetPointers(ours.matA, d["off"], d["col"], ours.a_val)
    n0 = native_count(on)
    try:
        want = theirs.compute(1.0, 0.0).clone()
    except cs.CuSparseError as e:                                        # the closed library refuses the class: so must we
        with pytest.raises(cs.CuSparseError) as mine:
            ours.compute(1.0, 0.0)
        assert mine.value.status == e.status
    else:
        assert torch.equal(ours.compute(1.0, 0.0), want)
    assert native_count(on) == n0
    ours.close(); theirs.close()


def test_recreated_descriptor_does_not_inherit_a_plan(cs, on, api):
    """A descriptor destroyed after a native run and one created next (the closed library may hand back the same address): the
    new one, set up in the default mode, never runs on the old plan."""
    A = csr(40, 40, np.random.default_rng(6).integers(0, 5, 40), 16, values="uniform")
    first = cs.SpGEMMReuse(on, dev(A, torch.float64), dev(A, torch.float64))
    n0 = native_count(on)
    first.compute()
    assert native_count(on) == n0 + 1
    old = first.desc.value
    first.close()
    on.set_option("B200SPMV_SPGEMM", "auto")
    second = cs.SpGEMMReuse(api, dev(A, torch.float64), dev(A, torch.float64))
    on.set_option("B200SPMV_SPGEMM", "on")
    n1 = native_count(on)
    second.compute()
    assert native_count(on) == n1, ("address reused" if second.desc.value == old else "new address")
    second.close()


# ---------------------------------------------------------------------------------------------------- the native entry points
def test_plan_refuses_bad_patterns_and_compute_counts_missing_products(cs, on):
    """b200spgemm_plan reports unsorted / out-of-range C columns, bad C offsets and out-of-range A columns without reading past
    them; on a C pattern that misses a column, compute skips and counts the missing products and writes the rest."""
    L = on.lib
    d = lambda a, dt=torch.int32: torch.tensor(a, dtype=dt, device="cuda")       # noqa: E731
    st = torch.cuda.current_stream().cuda_stream
    a_off, a_col = d([0, 2, 3]), d([0, 1, 1])
    b_off, b_col = d([0, 2, 3]), d([0, 2, 1])
    plan = torch.empty(L.b200spgemm_plan_size(2, 3, 3, 4) + 4096, dtype=torch.uint8, device="cuda")
    passes, bad = C.c_int64(-1), C.c_uint64(0)

    def run(c_off, c_col, nnz_c, a_c=a_col):
        return L.b200spgemm_plan(st, 2, 2, 3, 3, 3, nnz_c, a_off.data_ptr(), a_c.data_ptr(), 0, b_off.data_ptr(), 0, c_off.data_ptr(),
                                 c_col.data_ptr(), 0, plan.data_ptr(), plan.numel(), C.byref(passes), C.byref(bad))
    assert run(d([0, 3, 4]), d([0, 2, 1, 1]), 4) == -2 and bad.value & 2          # C row 0 unsorted
    assert run(d([0, 3, 4]), d([0, 1, 7, 1]), 4) == -2 and bad.value & 2          # C column out of range
    assert run(d([0, 5, 4]), d([0, 1, 2, 1]), 4) == -2 and bad.value & 1          # C offsets decrease / leave [0, nnz]
    assert run(d([0, 3, 4]), d([0, 1, 2, 1]), 4, d([0, 9, 1])) == -2 and bad.value & 4   # A column past B's rows
    # C row 0 lacks column 2: the product a_00 * b_02 is skipped and counted
    c_off, c_col = d([0, 2, 3]), d([0, 1, 1])
    assert run(c_off, c_col, 3) == 0 and bad.value == 0 and passes.value == 2
    a_val, b_val = d([2.0, 3.0, 5.0], torch.float64), d([7.0, 11.0, 13.0], torch.float64)
    c_val = torch.full((3,), float("nan"), dtype=torch.float64, device="cuda")
    one, zero = C.c_double(1.0), C.c_double(0.0)
    rc = L.b200spgemm_compute(st, 1, 2, 3, a_off.data_ptr(), a_col.data_ptr(), a_val.data_ptr(), 0, b_off.data_ptr(), b_col.data_ptr(),
                              b_val.data_ptr(), 0, c_off.data_ptr(), c_col.data_ptr(), c_val.data_ptr(), 0, C.addressof(one),
                              C.addressof(zero), 0, plan.data_ptr())
    torch.cuda.synchronize()
    assert rc == 0 and c_val.tolist() == [14.0, 39.0, 65.0]
    assert int(plan[8:16].view(torch.int64).item()) == 1


# ---------------------------------------------------------------------------------------------------- samples
def clean_env(**extra):
    env = {k: v for k, v in os.environ.items() if k != "B200SPMV_CUSPARSE"}
    env.update(extra)
    return env


def test_reuse_sample_computes_natively():
    exe = os.path.join(ROOT, "oracle", "_ref", "spgemm_reuse_example.b200")
    if not os.path.exists(exe):
        pytest.skip("oracle/_ref not built")
    p = subprocess.run([exe], capture_output=True, text=True, timeout=300, env=clean_env(B200SPMV_LOG="1", B200SPMV_SPGEMM="on"))
    assert p.returncode == 0 and "spgemm_reuse_example test PASSED" in p.stdout, p.stdout + p.stderr
    lines = [l for l in p.stderr.splitlines() if "SpGEMMreuse" in l]
    assert sum("compute native" in l for l in lines) == 2 and any("copy plan" in l for l in lines), lines
    assert not any("forwarded" in l for l in lines), lines


@pytest.mark.parametrize("name", ["spgemm_reuse", "spgemm", "spgemm_mem"])
def test_samples_pass_as_their_closed_builds(name):
    exe = os.path.join(ROOT, "oracle", "_ref", f"{name}_example")
    if not (os.path.exists(exe + ".b200") and os.path.exists(exe + ".cusparse")):
        pytest.skip("oracle/_ref not built")
    want = subprocess.run([exe + ".cusparse"], capture_output=True, text=True, timeout=300, env=clean_env())
    got = subprocess.run([exe + ".b200"], capture_output=True, text=True, timeout=300, env=clean_env())
    assert want.returncode == 0 and "PASSED" in want.stdout, want.stdout
    assert got.returncode == 0 and got.stdout == want.stdout, got.stdout + got.stderr
