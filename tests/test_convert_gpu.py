"""GPU: the format conversions of convert.cu -- csr2csc against scipy bit for bit at every value width, coosort against np.lexsort,
coo2csr / csr2coo / the identity permutation against numpy, all of them against the closed library through the shim (with the
shim's native / forwarded counts), determinism over stale workspaces and graph replays, canaries around every output for in-range and
out-of-range indices, and the coosort reference sample linked against the shim."""
import os
import re
import subprocess

import numpy as np
import pytest
import torch

from oracle import convert_ref as R
from oracle import oracle as O

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSR2CSC, ROW, COL, COO2CSR, CSR2COO, IDENTITY = range(6)
CANARY = 0x5C


@pytest.fixture(scope="module")
def L():
    if not torch.cuda.is_available():
        pytest.skip("no GPU")
    from cudalibrarysamples_b200 import lib
    return lib.shim()


def dev(a, dtype=torch.int32):
    return torch.tensor(np.asarray(a), device="cuda", dtype=dtype)


def stream():
    return torch.cuda.current_stream().cuda_stream


def random_bits(nnz, width, seed):
    """nnz values of `width` bytes with random bits (NaN payloads among them), as a (nnz, width) uint8 tensor"""
    rng = np.random.default_rng(seed)
    return torch.tensor(rng.integers(0, 256, (nnz, width), dtype=np.uint8), device="cuda")


def _random(rows, cols, nnz, seed):
    rng = np.random.default_rng(seed)
    flat = np.sort(rng.choice(rows * cols, nnz, replace=False))
    row, col = flat // cols, flat % cols
    return np.concatenate([[0], np.cumsum(np.bincount(row, minlength=rows))]), col


def _duplicates(rows, cols, nnz, seed):
    """repeated (row, col) entries, columns unsorted within each row"""
    rng = np.random.default_rng(seed)
    row = np.sort(rng.integers(0, rows, nnz))
    return np.concatenate([[0], np.cumsum(np.bincount(row, minlength=rows))]), rng.integers(0, cols, nnz)


def patterns():
    off, col, _ = O.rmat_csr(1 << 14, avg_nnz=16, seed=3, val_seed=4)                # hub columns
    yield "rmat", off, col, 1 << 14, 1 << 14
    off, col, _ = O.rmat_csr(3000, cols=70000, avg_nnz=8, seed=5, val_seed=6)         # three radix passes
    yield "rmat_wide", off, col, 3000, 70000
    off, col, _ = O.gen_stencil5(61)
    yield "stencil5", off, col, len(off) - 1, len(off) - 1
    yield "empty_rows_and_cols", *_random(500, 400, 600, 1), 500, 400
    yield "duplicates_unsorted", *_duplicates(777, 45, 9000, 2), 777, 45
    yield "no_entries", np.zeros(9, np.int64), np.zeros(0, np.int64), 8, 5
    yield "no_rows", np.zeros(1, np.int64), np.zeros(0, np.int64), 0, 5
    yield "no_cols", np.zeros(4, np.int64), np.zeros(0, np.int64), 3, 0


def run_csr2csc(L, m, n, off, col, vals, width, base, fill=0):
    """b200csr2csc on fresh outputs and a workspace filled with `fill`; returns (ptr, ind, val bytes)"""
    nnz = col.numel()
    ptr = torch.full((n + 1,), -7, dtype=torch.int32, device="cuda")
    ind = torch.full((max(nnz, 1),), -7, dtype=torch.int32, device="cuda")
    out = None if vals is None else torch.full_like(vals, 0xEE)
    wsb = L.b200csr2csc_workspace_bytes(m, n, nnz)
    ws = torch.full((max(wsb, 16),), fill, dtype=torch.uint8, device="cuda")
    rc = L.b200csr2csc(stream(), m, n, nnz, None if vals is None else vals.data_ptr(), off.data_ptr(), col.data_ptr() if nnz else None,
                       None if out is None else out.data_ptr(), ptr.data_ptr(), ind.data_ptr(), width, int(vals is not None), base,
                       ws.data_ptr(), wsb)
    torch.cuda.synchronize()
    assert rc == 0
    return ptr, ind[:nnz], out


@pytest.mark.parametrize("base", [0, 1])
def test_csr2csc_matches_scipy_bit_for_bit(L, base):
    for name, off, col, m, n in patterns():
        offd, cold = dev(np.asarray(off) + base), dev(np.asarray(col) + base)
        want_ptr, want_ind, _ = R.csr2csc(np.asarray(off) + base, np.asarray(col) + base, None, m, n, base)
        _, _, perm = R.T.plan_scipy(np.asarray(off) + base, np.asarray(col) + base, m, n, base)
        for width in (0, 1, 2, 4, 8, 16):                   # 0: SYMBOLIC
            vals = None if width == 0 else random_bits(len(col), width, 9)
            ptr, ind, out = run_csr2csc(L, m, n, offd, cold, vals, width, base)
            assert ptr.tolist() == want_ptr.tolist() and ind.tolist() == want_ind.tolist(), (name, width)
            if vals is not None:
                assert torch.equal(out, vals[torch.as_tensor(perm, device="cuda")]), (name, width)


def test_csr2csc_is_deterministic_over_stale_workspaces_and_graph_replays(L):
    off, col, _ = O.rmat_csr(1 << 14, avg_nnz=16, seed=11, val_seed=12)
    m = n = 1 << 14
    offd, cold = dev(off), dev(col)
    vals = random_bits(len(col), 8, 1).view(torch.int64).reshape(-1)
    runs = [run_csr2csc(L, m, n, offd, cold, vals, 8, 0, fill) for fill in (0x00, 0x7F, 0x00)]
    for r in runs[1:]:
        assert all(torch.equal(a, b) for a, b in zip(runs[0], r))
    # captured once, replayed with new values in the same input buffer
    nnz = len(col)
    ptr, ind, out = (torch.empty(n + 1, dtype=torch.int32, device="cuda"), torch.empty(nnz, dtype=torch.int32, device="cuda"),
                     torch.empty_like(vals))
    src = vals.clone()
    wsb = L.b200csr2csc_workspace_bytes(m, n, nnz)
    ws = torch.full((wsb,), 0x7F, dtype=torch.uint8, device="cuda")
    s = torch.cuda.Stream()
    g = torch.cuda.CUDAGraph()
    torch.cuda.synchronize()
    with torch.cuda.graph(g, stream=s):
        rc = L.b200csr2csc(s.cuda_stream, m, n, nnz, src.data_ptr(), offd.data_ptr(), cold.data_ptr(), out.data_ptr(), ptr.data_ptr(),
                           ind.data_ptr(), 8, 1, 0, ws.data_ptr(), wsb)
    assert rc == 0
    for seed in (2, 3):
        src.copy_(random_bits(nnz, 8, seed).view(torch.int64).reshape(-1))
        g.replay()
        torch.cuda.synchronize()
        want = run_csr2csc(L, m, n, offd, cold, src, 8, 0)
        assert torch.equal(ptr, want[0]) and torch.equal(ind, want[1]) and torch.equal(out, want[2])


def canaried(n, dtype=torch.int32, pad=64):
    """a view of n elements inside an allocation whose pad elements on either side hold the canary byte"""
    esz = torch.empty(0, dtype=dtype).element_size()
    raw = torch.full(((n + 2 * pad) * esz,), CANARY, dtype=torch.uint8, device="cuda")
    return raw, raw[pad * esz:(pad + n) * esz].view(dtype)


def intact(raw, n, dtype=torch.int32, pad=64):
    esz = torch.empty(0, dtype=dtype).element_size()
    return bool((raw[:pad * esz] == CANARY).all()) and bool((raw[(pad + n) * esz:] == CANARY).all())


@pytest.mark.parametrize("bad", ["in_range", "large", "negative", "past_n"])
def test_outputs_and_workspaces_keep_their_canaries(L, bad):
    m, n = 3000, 70000
    off, col, _ = O.rmat_csr(m, cols=n, avg_nnz=8, seed=5, val_seed=6)
    col = np.asarray(col, np.int64)
    rng = np.random.default_rng(4)
    hit = rng.choice(col.size, 40, replace=False)
    col[hit] = {"in_range": col[hit], "large": 2 ** 31 - 1 - rng.integers(0, 5, 40), "negative": -rng.integers(1, 2 ** 31 - 1, 40),
                "past_n": n + rng.integers(0, 300, 40)}[bad]
    nnz = col.size
    offd, cold = dev(off), dev(col)
    vals = random_bits(nnz, 16, 3)
    # csr2csc
    rp, ptr = canaried(n + 1)
    ri, ind = canaried(nnz)
    rv, out = canaried(nnz * 16, torch.uint8)
    wsb = L.b200csr2csc_workspace_bytes(m, n, nnz)
    rw, ws = canaried(wsb // 8, torch.int64, 16)                  # 16-byte aligned workspace of exactly wsb bytes (wsb % 256 == 0)
    assert L.b200csr2csc(stream(), m, n, nnz, vals.data_ptr(), offd.data_ptr(), cold.data_ptr(), out.data_ptr(), ptr.data_ptr(),
                         ind.data_ptr(), 16, 1, 0, ws.data_ptr(), wsb) == 0
    torch.cuda.synchronize()
    assert intact(rp, n + 1) and intact(ri, nnz) and intact(rv, nnz * 16, torch.uint8) and intact(rw, wsb // 8, torch.int64, 16)
    # coosort on the same indices as COO (row keys in range, column keys as above), both orders
    for by_row in (1, 0):
        rr, rows = canaried(nnz)
        rc_, cols = canaried(nnz)
        rP, P = canaried(nnz)
        rows.copy_(dev(R.csr2coo(off)))
        cols.copy_(cold)
        P.copy_(torch.arange(nnz, dtype=torch.int32, device="cuda"))
        wsb = L.b200coosort_workspace_bytes(m, n, nnz)
        rw, ws = canaried(wsb // 8, torch.int64, 16)
        assert L.b200coosort(stream(), by_row, m, n, nnz, rows.data_ptr(), cols.data_ptr(), P.data_ptr(), ws.data_ptr(), wsb) == 0
        torch.cuda.synchronize()
        assert intact(rr, nnz) and intact(rc_, nnz) and intact(rP, nnz) and intact(rw, wsb // 8, torch.int64, 16), by_row
        assert sorted(P.tolist()) == list(range(nnz))               # a permutation whatever the keys
    # coo2csr with the bad keys as row indices, csr2coo with offsets that run past nnz
    ro, offs = canaried(n + 1)
    assert L.b200coo2csr(stream(), cold.data_ptr(), nnz, n, offs.data_ptr(), 0) == 0
    bad_off = offd.clone()
    bad_off[len(off) // 2] = 2 ** 31 - 1
    rr, rows = canaried(nnz)
    assert L.b200csr2coo(stream(), bad_off.data_ptr(), nnz, m, rows.data_ptr(), 0) == 0
    torch.cuda.synchronize()
    assert intact(ro, n + 1) and intact(rr, nnz)


def coo_inputs():
    rng = np.random.default_rng(21)
    m, n = 1000, 777                                                  # not powers of two
    r, c = rng.integers(0, m, 20000), rng.integers(0, n, 20000)     # duplicates among them
    yield "random", m, n, r, c
    o = np.lexsort((c, r))
    yield "sorted", m, n, r[o], c[o]
    yield "reversed", m, n, r[o][::-1].copy(), c[o][::-1].copy()
    yield "base1_keys_to_m", m, n, r + 1, c + 1                        # keys 1 .. m / 1 .. n
    yield "wide_keys", 70000, 3, rng.integers(0, 70001, 5000), rng.integers(0, 4, 5000)
    yield "one", 5, 5, np.array([4]), np.array([2])
    yield "none", 5, 5, np.zeros(0, np.int64), np.zeros(0, np.int64)


def run_coosort(L, by_row, m, n, r, c, P):
    nnz = len(r)
    rows, cols, Pd = dev(r), dev(c), dev(P)
    wsb = L.b200coosort_workspace_bytes(m, n, nnz)
    ws = torch.full((max(wsb, 16),), 0x7F, dtype=torch.uint8, device="cuda")
    if nnz:
        assert L.b200coosort(stream(), by_row, m, n, nnz, rows.data_ptr(), cols.data_ptr(), Pd.data_ptr(), ws.data_ptr(), wsb) == 0
    torch.cuda.synchronize()
    return rows.cpu().numpy(), cols.cpu().numpy(), Pd.cpu().numpy()


@pytest.mark.parametrize("by_row", [1, 0])
def test_coosort_matches_lexsort(L, by_row):
    rng = np.random.default_rng(5)
    for name, m, n, r, c in coo_inputs():
        for P in (np.arange(len(r)), rng.permutation(len(r)) * 3 + 1):     # identity and a non-identity P
            got = run_coosort(L, by_row, m, n, r, c, P)
            want = R.coosort(r, c, P, bool(by_row))
            for g, w, what in zip(got, want, ("rows", "cols", "P")):
                assert np.array_equal(g, w), (name, what)


def test_coo2csr_csr2coo_identity_match_numpy(L):
    for name, off, col, m, n in patterns():
        for base in (0, 1):
            offd = dev(np.asarray(off) + base)
            nnz = len(col)
            rows = torch.full((max(nnz, 1),), -1, dtype=torch.int32, device="cuda")
            assert L.b200csr2coo(stream(), offd.data_ptr(), nnz, m, rows.data_ptr(), base) == 0
            back = torch.full((m + 1,), -1, dtype=torch.int32, device="cuda")
            assert L.b200coo2csr(stream(), rows.data_ptr(), nnz, m, back.data_ptr(), base) == 0
            torch.cuda.synchronize()
            assert rows[:nnz].tolist() == R.csr2coo(np.asarray(off) + base, base).tolist(), name
            assert back.tolist() == (np.asarray(off) + base).tolist(), name
    for k in (0, 1, 1000, 1 << 20):
        p = torch.full((max(k, 1),), -1, dtype=torch.int32, device="cuda")
        assert L.b200identity_permutation(stream(), k, p.data_ptr()) == 0
        torch.cuda.synchronize()
        assert torch.equal(p[:k], torch.arange(k, dtype=torch.int32, device="cuda"))


# ------------------------------------------------------------------------------------------ through the shim, against the closed library
def apis():
    from cudalibrarysamples_b200 import cusparse_api as cs
    return cs, cs.Api("b200"), cs.Api("cusparse")


def expect_counts(api, st_native):
    s = api.stats()
    assert (s["native"], s["forwarded"]) == ((1, 0) if st_native else (0, 1)), s


def test_csr2csc_through_the_shim_equals_the_closed_library(L):
    cs, ours, closed = apis()
    for name, off, col, m, n in patterns():
        if name == "duplicates_unsorted" or len(col) == 0:
            continue
        for base in (0, 1):
            offd, cold = dev(np.asarray(off) + base), dev(np.asarray(col) + base)
            for dt in (None, torch.float16, torch.float32, torch.float64, torch.complex128):
                vals = None if dt is None else random_bits(len(col), torch.empty(0, dtype=dt).element_size(), 4).view(dt).reshape(-1)
                ours.reset_stats()
                a = cs.csr2csc(ours, m, n, offd, cold, vals, base)
                width = 0 if dt is None else vals.element_size()
                routed = L.b200conv_route(CSR2CSC, m, n, len(col), width, 1, 256)
                expect_counts(ours, routed)
                b = cs.csr2csc(closed, m, n, offd, cold, vals, base)
                for x, y, what in zip(a, b, ("ptr", "ind", "val")):
                    assert (x is None and y is None) or torch.equal(x.view(torch.uint8), y.view(torch.uint8)), (name, base, dt, what)


def test_coosort_coo2csr_csr2coo_through_the_shim_equal_the_closed_library(L, capsys):
    cs, ours, closed = apis()
    rng = np.random.default_rng(8)
    # the last shape is in the routed class
    for m, n, nnz in ((1000, 777, 20000), (70000, 300, 30000), (5, 5, 1), (1 << 20, 1 << 20, 4 << 20)):
        flat = rng.permutation(np.unique(rng.integers(0, m * n, nnz + nnz // 8 + 8)))[:nnz]      # duplicate-free, shuffled
        r, c = flat // n, flat % n
        P = rng.permutation(nnz).astype(np.int32)
        for by_row in (True, False):
            res = []
            for api in (ours, closed):
                api.reset_stats()
                rows, cols, Pd = dev(r), dev(c), dev(P)
                cs.coosort(api, m, n, rows, cols, Pd, by_row)
                res.append((rows, cols, Pd))
                if api is ours:                     # the closed Api's reset clears the same counters
                    expect_counts(ours, L.b200conv_route(ROW if by_row else COL, m, n, nnz, 0, 0, 256))
            for x, y, what in zip(*res, ("rows", "cols", "P")):
                assert torch.equal(x, y), (m, n, by_row, what)
            want = R.coosort(r, c, P, by_row)
            assert np.array_equal(res[1][2].cpu().numpy(), want[2])      # the closed library composes P as P_in[sigma]
        # the identity permutation, and P created by cusparseCreateIdentityPermutation
        rows, cols = dev(r), dev(c)
        ours.reset_stats()
        Pa = cs.coosort(ours, m, n, rows, cols, None, True)
        s = ours.stats()
        routed = L.b200conv_route(IDENTITY, 0, 0, nnz, 0, 0, None) + L.b200conv_route(ROW, m, n, nnz, 0, 0, 256)
        assert (s["native"], s["forwarded"]) == (routed, 2 - routed), s
        assert np.array_equal(Pa.cpu().numpy(), R.coosort(r, c)[2])
        # coo2csr / csr2coo on the sorted rows
        srt = np.sort(r)
        offs = [cs.coo2csr(api, dev(srt), m) for api in (ours, closed)]
        assert torch.equal(offs[0], offs[1]) and offs[0].tolist() == R.coo2csr(srt, m).tolist()
        coos = [cs.csr2coo(api, offs[1], nnz) for api in (ours, closed)]
        assert torch.equal(coos[0], coos[1]) and coos[0].tolist() == srt.tolist()
    # with duplicate pairs: is the closed library's sort stable?  (DESIGN.md 3.23 records the answer; ours is)
    r, c = rng.integers(0, 50, 40000), rng.integers(0, 40, 40000)
    for by_row in (True, False):
        rows, cols, Pd = dev(r), dev(c), dev(np.arange(len(r)))
        cs.coosort(closed, 50, 40, rows, cols, Pd, by_row)
        stable = np.array_equal(Pd.cpu().numpy(), R.coosort(r, c, None, by_row)[2])
        with capsys.disabled():
            print(f"\nclosed coosort {'ByRow' if by_row else 'ByColumn'} with duplicates: {'stable' if stable else 'NOT stable'}")


def test_forward_env_forwards_every_conversion():
    """B200SPMV_FORWARD=1: the same calls all go to the closed library, counted"""
    code = r"""
import numpy as np, torch
from cudalibrarysamples_b200 import cusparse_api as cs
api = cs.Api("b200")
api.reset_stats()
off = torch.tensor([0, 2, 3, 5], dtype=torch.int32, device="cuda")
col = torch.tensor([1, 0, 2, 0, 1], dtype=torch.int32, device="cuda")
cs.csr2csc(api, 3, 3, off, col, torch.arange(5, dtype=torch.float32, device="cuda"))
rows = cs.csr2coo(api, off, 5)
cs.coo2csr(api, rows, 3)
cs.coosort(api, 3, 3, rows.clone(), col.clone(), None, False)
s = api.stats()
assert (s["native"], s["forwarded"]) == (0, 5), s
print("OK")
"""
    env = dict(os.environ, B200SPMV_FORWARD="1")
    p = subprocess.run(["python", "-c", code], capture_output=True, text=True, cwd=ROOT, env=env, timeout=600)
    assert p.returncode == 0 and p.stdout.strip().endswith("OK"), p.stdout + p.stderr


def test_reference_sample_passes_on_the_shim(L):
    exe = os.path.join(ROOT, "oracle", "_ref", "coosort_example.b200")
    if not os.path.exists(exe):
        pytest.skip("oracle/_ref not built (needs the reference checkout at build time)")
    p = subprocess.run([exe], capture_output=True, text=True, env=dict(os.environ, B200SPMV_LOG="1"), timeout=300)
    assert p.returncode == 0 and "PASSED" in p.stdout, p.stdout + p.stderr
    verdict = re.findall(r"\[b200spmv\] XcoosortByRow (native|forwarded)", p.stderr)
    assert verdict == ["native" if L.b200conv_route(ROW, 4, 4, 11, 0, 0, 256) else "forwarded"], p.stderr
