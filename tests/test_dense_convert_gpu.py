"""GPU: sparse <-> dense conversion (dense_convert.cu) -- every native entry point bit-identical to oracle/dense_ref.py at every
width, order and base, with ld padding, canaries, odd ld and an offset dense pointer; against the closed library through the shim
(with the route's native / forwarded counts); the closed library's zero predicate, duplicate and -1-slot behaviour printed and
matched; graph replay; the nnz refresh of cusparseCsrSetPointers; the three reference samples linked against the shim."""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pytest
import torch

from oracle import dense_ref as R

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
COL, ROW = R.ORDER_COL, R.ORDER_ROW
CANARY = 0xA5
PAD = 64                                   # canary bytes on either side of every output
# value type per width for the dense -> sparse predicate (cudaDataType) and its part width
VT = {2: (2, 2), 4: (0, 4), 8: (1, 8), 16: (5, 8)}     # fp16, fp32, fp64, complex128
TORCH = {2: torch.float16, 4: torch.float32, 8: torch.float64, 16: torch.complex128}


@pytest.fixture(scope="module")
def L():
    if not torch.cuda.is_available():
        pytest.skip("no GPU")
    from cudalibrarysamples_b200 import lib
    return lib.shim()


def stream():
    return torch.cuda.current_stream().cuda_stream


def canaried(nbytes, shift=0):
    """(raw, view): nbytes at raw[PAD + shift:], PAD canary bytes on either side"""
    raw = torch.full((nbytes + 2 * PAD + shift,), CANARY, dtype=torch.uint8, device="cuda")
    return raw, raw[PAD + shift:PAD + shift + nbytes]


def intact(raw, nbytes, shift=0):
    return bool((raw[:PAD + shift] == CANARY).all()) and bool((raw[PAD + shift + nbytes:] == CANARY).all())


def dev(a, dtype=torch.int32):
    return torch.tensor(np.asarray(a), device="cuda", dtype=dtype)


def random_csr(rng, m, n, density, base, dup=False):
    nnz_row = rng.binomial(n, density, m)
    if m > 4:
        nnz_row[m // 3] = n                          # one full row: longer than a warp's chunk and a CTA panel
    cols = [np.sort(rng.choice(n, k, replace=False)) for k in nnz_row]
    if dup:
        cols = [np.concatenate([c, rng.choice(c, len(c) // 2)]) if len(c) else c for c in cols]
    off = np.concatenate([[0], np.cumsum([len(c) for c in cols])])
    ind = np.concatenate(cols) if cols else np.zeros(0, np.int64)
    return off + base, ind.astype(np.int64) + base


def vals_bits(rng, nnz, w, zeros=False):
    v = rng.integers(0, 256, (nnz, w), dtype=np.uint8)
    if zeros and nnz:
        v[rng.random(nnz) < 0.3] = 0                 # explicit zeros among the values
    return v


def dense_bytes(m, n, ld, order, w):
    return (m * ld if order == ROW else n * ld) * w if m and n else 0


SHAPES = [(1, 1), (5, 4), (37, 61), (70, 1300), (1300, 70), (0, 5), (5, 0)]


@pytest.mark.parametrize("w", [2, 4, 8, 16])
def test_csr_csc_to_dense_bit_exact_with_canaries(L, w):
    rng = np.random.default_rng(w)
    for m, n in SHAPES:
        for csc in (0, 1):
            for order in (ROW, COL):
                for base in (0, 1):
                    for pad_ld, shift in ((0, 0), (3, 0), (1, w)):   # tight; ld padding; odd ld with the pointer one element on
                        M, N = (n, m) if csc else (m, n)
                        off, ind = random_csr(rng, M, N, 0.2, base, dup=(m == 37))
                        nnz = len(ind)
                        vals = vals_bits(rng, nnz, w)
                        ld = max(1, (n if order == ROW else m) + pad_ld)
                        nb = dense_bytes(m, n, ld, order, w)
                        raw, d = canaried(nb, shift)
                        init = rng.integers(0, 256, nb, dtype=np.uint8)
                        d.copy_(torch.from_numpy(init).cuda())
                        offd, indd, vd = dev(off), dev(ind if nnz else [0]), torch.from_numpy(vals.reshape(-1) if nnz else np.zeros(w, np.uint8)).cuda()
                        rc = L.b200csr2dense(stream(), csc, m, n, nnz, offd.data_ptr(), indd.data_ptr(), vd.data_ptr(), w, base,
                                             d.data_ptr(), ld, order)
                        torch.cuda.synchronize()
                        assert rc == 0
                        want = R.csr_to_dense(init.reshape(-1, w), m, n, ld, order, off, ind, vals, base, bool(csc))
                        got = d.cpu().numpy().reshape(-1, w)
                        assert np.array_equal(got, want), (m, n, csc, order, base, pad_ld)
                        assert intact(raw, nb, shift), (m, n, csc, order, base, pad_ld)


@pytest.mark.parametrize("w", [2, 4, 8, 16])
def test_dense_to_csr_csc_bit_exact_with_canaries(L, w):
    rng = np.random.default_rng(10 + w)
    vt, part = VT[w]
    for m, n in SHAPES:
        for csc in (0, 1):
            for order in (ROW, COL):
                for base in (0, 1):
                    for pad_ld, shift in ((0, 0), (3, 0), (1, w)):
                        ld = max(1, (n if order == ROW else m) + pad_ld)
                        nb = dense_bytes(m, n, ld, order, w)
                        init = vals_bits(rng, nb // w, w, zeros=True)
                        init[rng.random(nb // w) < 0.6] = 0
                        init[rng.random(nb // w) < 0.05, -1] = 0x80          # -0 / negative parts
                        off, ind, vals = R.dense_to_csr(init, m, n, ld, order, part, base, bool(csc))
                        nnz = len(ind)
                        raw_d, d = canaried(nb, shift)
                        d.copy_(torch.from_numpy(init.reshape(-1)).cuda())
                        raw_i, di = canaried(nnz * 4)
                        raw_v, dv = canaried(nnz * w)
                        offd = dev(off)
                        rc = L.b200dense2csr(stream(), csc, m, n, nnz, d.data_ptr(), ld, order, vt, offd.data_ptr(), di.data_ptr(),
                                             dv.data_ptr(), base)
                        torch.cuda.synchronize()
                        assert rc == 0
                        assert np.array_equal(di.cpu().numpy().view(np.int32), ind), (m, n, csc, order, base, pad_ld)
                        assert np.array_equal(dv.cpu().numpy().reshape(-1, w), vals.reshape(-1, w)), (m, n, csc, order, base)
                        assert intact(raw_i, nnz * 4) and intact(raw_v, nnz * w) and intact(raw_d, nb, shift)


def test_dense_to_csr_never_writes_outside_its_offsets(L):
    """A changed since the analysis: rows with more non-zeros than their range keep the first ones, rows with fewer leave the
    rest unwritten"""
    rng = np.random.default_rng(3)
    m, n, w = 300, 257, 4
    for order in (ROW, COL):
        A = np.where(rng.random((m, n)) < 0.3, rng.standard_normal((m, n)), 0).astype(np.float32)
        off, ind, vals = R.dense_to_csr(A.view(np.uint8).reshape(-1, 4) if order == ROW else A.T.copy().view(np.uint8).reshape(-1, 4),
                                        m, n, n if order == ROW else m, order, 4)
        B = A.copy()
        B[::2] = rng.standard_normal((len(B[::2]), n))               # denser than analysed
        B[1::2] = 0                                                 # emptier than analysed
        flat = B if order == ROW else B.T.copy()
        nnz = len(ind)
        raw_i, di = canaried(nnz * 4)
        raw_v, dv = canaried(nnz * w)
        d = torch.from_numpy(flat.reshape(-1).copy()).cuda()
        rc = L.b200dense2csr(stream(), 0, m, n, nnz, d.data_ptr(), n if order == ROW else m, order, 0, dev(off).data_ptr(),
                             di.data_ptr(), dv.data_ptr(), 0)
        torch.cuda.synchronize()
        assert rc == 0 and intact(raw_i, nnz * 4) and intact(raw_v, nnz * w)
        gi = di.cpu().numpy().view(np.int32)
        for r in range(0, m, 2):
            k = off[r + 1] - off[r]
            assert gi[off[r]:off[r + 1]].tolist() == list(range(k)), r          # the first k columns of a full row
        for r in range(1, m, 2):
            assert (di.cpu().numpy()[off[r] * 4:off[r + 1] * 4] == CANARY).all(), r   # unwritten


@pytest.mark.parametrize("w", [2, 4, 8, 16])
def test_coo_and_blocked_ell_to_dense_bit_exact(L, w):
    rng = np.random.default_rng(20 + w)
    for m, n, bs in ((4, 6, 2), (64, 96, 16), (70, 50, 32), (128, 128, 64)):
        for order in (ROW, COL):
            for base in (0, 1):
                ld = (n if order == ROW else m) + 1
                nb = dense_bytes(m, n, ld, order, w)
                init = rng.integers(0, 256, nb, dtype=np.uint8)
                # COO, unsorted, no duplicates
                flat = rng.choice(m * n, m * n // 7, replace=False)
                r, c = flat // n, flat % n
                vals = vals_bits(rng, len(r), w)
                raw, d = canaried(nb)
                d.copy_(torch.from_numpy(init).cuda())
                assert L.b200coo2dense(stream(), m, n, len(r), dev(r + base).data_ptr(), dev(c + base).data_ptr(),
                                       torch.from_numpy(vals.reshape(-1)).cuda().data_ptr(), w, base, d.data_ptr(), ld, order) == 0
                torch.cuda.synchronize()
                assert np.array_equal(d.cpu().numpy().reshape(-1, w), R.scatter(init.reshape(-1, w), m, n, ld, order, r, c, vals))
                assert intact(raw, nb)
                # Blocked-ELL with -1 padding holding NaN-like bits
                nbr, nbc = (m + bs - 1) // bs, (n + bs - 1) // bs
                slots = max(1, nbc // 2)
                colind = np.full((nbr, slots), -1, np.int64)
                for br in range(nbr):
                    k = rng.integers(0, slots + 1)
                    colind[br, :k] = np.sort(rng.choice(nbc, k, replace=False))
                ev = vals_bits(rng, m * slots * bs, w)
                ev[:, -1] |= 0x7F
                raw, d = canaried(nb)
                d.copy_(torch.from_numpy(init).cuda())
                ci = np.where(colind >= 0, colind + base, -1)
                assert L.b200bell2dense(stream(), m, n, bs, slots * bs, dev(ci).data_ptr(), torch.from_numpy(ev.reshape(-1)).cuda().data_ptr(),
                                        w, base, d.data_ptr(), ld, order) == 0
                torch.cuda.synchronize()
                assert np.array_equal(d.cpu().numpy().reshape(-1, w), R.bell_to_dense(init.reshape(-1, w), m, n, ld, order, bs, ci, ev, base))
                assert intact(raw, nb)
                # and back: dense -> Blocked-ELL on the same colind, NaN-prefilled values
                src = rng.integers(0, 256, nb, dtype=np.uint8)
                raw, out = canaried(m * slots * bs * w)
                out.fill_(0xFF)
                assert L.b200dense2bell(stream(), m, n, bs, slots * bs, torch.from_numpy(src).cuda().data_ptr(), ld, order, w,
                                        dev(ci).data_ptr(), out.data_ptr(), base) == 0
                torch.cuda.synchronize()
                want = R.dense_to_bell(src.reshape(-1, w), m, n, ld, order, bs, ci, np.full((m * slots * bs, w), 0xFF, np.uint8), base)
                assert np.array_equal(out.cpu().numpy().reshape(-1, w), want) and intact(raw, m * slots * bs * w)


def test_rejects_bad_arguments(L):
    d = torch.zeros(64, dtype=torch.float32, device="cuda")
    off = torch.zeros(9, dtype=torch.int32, device="cuda")
    p = d.data_ptr()
    assert L.b200csr2dense(stream(), 0, 4, 4, 0, off.data_ptr(), None, None, 3, 0, p, 4, ROW) == -1       # width
    assert L.b200csr2dense(stream(), 0, 4, 4, 0, off.data_ptr(), None, None, 4, 2, p, 4, ROW) == -1       # base
    assert L.b200csr2dense(stream(), 0, 4, 4, 0, off.data_ptr(), None, None, 4, 0, p, 3, ROW) == -1       # ld
    assert L.b200csr2dense(stream(), 0, 4, 4, 0, off.data_ptr(), None, None, 4, 0, p, 4, 3) == -1         # order
    assert L.b200csr2dense(stream(), 0, 4, 4, 1, off.data_ptr(), None, None, 4, 0, p, 4, ROW) == -1       # NULL ind with nnz
    assert L.b200dense2csr(stream(), 0, 4, 4, 1, p, 4, ROW, 10, off.data_ptr(), p, p, 0) == -1            # integer type
    assert L.b200bell2dense(stream(), 4, 4, 2, 3, off.data_ptr(), p, 4, 0, p, 4, ROW) == -1               # ell_cols % bs
    assert L.b200csr2dense(stream(), 0, 4, 4, 0, off.data_ptr(), None, None, 4, 0, p, 4, ROW) == 0        # nnz = 0: zeros
    torch.cuda.synchronize()
    assert not d[:16].any()


def test_graph_replay_is_bit_identical(L):
    rng = np.random.default_rng(9)
    m, n = 2000, 3000
    off, ind = random_csr(rng, m, n, 0.01, 0)
    nnz = len(ind)
    vals = torch.from_numpy(vals_bits(rng, nnz, 8).reshape(-1)).cuda()
    offd, indd = dev(off), dev(ind)
    out = torch.empty(m * n * 8, dtype=torch.uint8, device="cuda")
    back_i, back_v = torch.empty(nnz, dtype=torch.int32, device="cuda"), torch.empty(nnz * 8, dtype=torch.uint8, device="cuda")
    s = torch.cuda.Stream()
    g = torch.cuda.CUDAGraph()
    torch.cuda.synchronize()
    with torch.cuda.graph(g, stream=s):
        assert L.b200csr2dense(s.cuda_stream, 0, m, n, nnz, offd.data_ptr(), indd.data_ptr(), vals.data_ptr(), 8, 0, out.data_ptr(), m, COL) == 0
        assert L.b200dense2csr(s.cuda_stream, 0, m, n, nnz, out.data_ptr(), m, COL, 1, offd.data_ptr(), back_i.data_ptr(),
                               back_v.data_ptr(), 0) == 0
    res = []
    for _ in range(2):
        out.fill_(7)
        g.replay()
        torch.cuda.synchronize()
        res.append((out.clone(), back_i.clone(), back_v.clone()))
    assert all(torch.equal(a, b) for a, b in zip(*res))
    nz = R.nonzero(vals.cpu().numpy().reshape(-1, 8), 8)
    want_i = ind[nz]
    assert np.array_equal(res[0][1].cpu().numpy()[:nz.sum()], want_i)


# ------------------------------------------------------------------------------------------ through the shim, against the closed library
def apis():
    from cudalibrarysamples_b200 import cusparse_api as cs
    return cs, cs.Api("b200"), cs.Api("cusparse")


def route(L, direction, fmt, order, vt, m, n, nnz, bs=0):
    return L.b200dense_route(direction, fmt, order, vt, 2, 2, 0, m, n, nnz, 1, 0, bs)


VTYPE = {torch.float16: 2, torch.bfloat16: 14, torch.float32: 0, torch.float64: 1, torch.complex64: 4, torch.complex128: 5}


@pytest.fixture(params=["auto", "on"])
def mode(request, L):
    """B200SPMV_DENSE: "auto" routes the measured classes only, "on" sends every admitted call to the native kernels, so the
    shim's own plumbing (getters, side table, ld, order) runs against the closed library"""
    assert L.b200spmv_set_option(b"B200SPMV_DENSE", request.param.encode()) == 0
    yield request.param
    assert L.b200spmv_set_option(b"B200SPMV_DENSE", b"auto") == 0


def expect_counts(ours, r):
    s = ours.stats()
    assert (s["native"], s["forwarded"]) == ((1, 0) if r else (0, 1)), s


def test_sparse_to_dense_native_and_shim_equal_the_closed_library(L, mode):
    """b200csr2dense (CSR and CSC) and b200coo2dense called directly, and cusparseSparseToDense through the shim, all bit-identical
    to the closed library's cusparseSparseToDense on the same inputs"""
    cs, ours, closed = apis()
    rng = np.random.default_rng(31)
    for m, n in ((5, 4), (300, 257), (1000, 3)):
        for dt in (torch.float16, torch.bfloat16, torch.float32, torch.float64, torch.complex128):
            w = torch.empty(0, dtype=dt).element_size()
            for fmt in (cs.CUSPARSE_FORMAT_CSR, cs.CUSPARSE_FORMAT_CSC, cs.CUSPARSE_FORMAT_COO):
                for order in (ROW, COL):
                    for base in (0, 1):
                        M, N = (n, m) if fmt == cs.CUSPARSE_FORMAT_CSC else (m, n)
                        off, ind = random_csr(rng, M, N, 0.1, base)
                        nnz = len(ind)
                        vals = torch.from_numpy(vals_bits(rng, nnz, w).reshape(-1)).cuda().view(dt)
                        if fmt == cs.CUSPARSE_FORMAT_COO:
                            a, b = dev(np.repeat(np.arange(M), np.diff(off)) + base), dev(ind)
                        else:
                            a, b = dev(off), dev(ind)
                        ld = (n if order == ROW else m) + 2
                        size = ld * (m if order == ROW else n)
                        fresh = lambda: torch.full((size * w,), 0x3C, dtype=torch.uint8, device="cuda").view(dt)  # noqa: E731
                        want = cs.sparse_to_dense(closed, fmt, m, n, a, b, vals, fresh(), ld, order, base).view(torch.uint8)
                        ours.reset_stats()
                        shim = cs.sparse_to_dense(ours, fmt, m, n, a, b, vals, fresh(), ld, order, base).view(torch.uint8)
                        expect_counts(ours, route(L, 0, fmt, order, VTYPE[dt], m, n, nnz))
                        native = fresh()
                        if fmt == cs.CUSPARSE_FORMAT_COO:
                            rc = L.b200coo2dense(stream(), m, n, nnz, a.data_ptr(), b.data_ptr(), vals.data_ptr(), w, base, native.data_ptr(),
                                                 ld, order)
                        else:
                            rc = L.b200csr2dense(stream(), int(fmt == cs.CUSPARSE_FORMAT_CSC), m, n, nnz, a.data_ptr(), b.data_ptr(),
                                                 vals.data_ptr(), w, base, native.data_ptr(), ld, order)
                        torch.cuda.synchronize()
                        assert rc == 0
                        case = (mode, m, n, dt, fmt, order, base)
                        assert torch.equal(native.view(torch.uint8), want), case
                        assert torch.equal(shim, want), case


def bell_pattern(rng, m, n, bs):
    """block columns of an m x n Blocked-ELL matrix, half the block columns per block row at most, -1 padding at every row's end
    (and one block row all padding)"""
    nbr, nbc = m // bs, n // bs
    slots = max(1, nbc // 2)
    colind = np.full((nbr, slots), -1, np.int64)
    for br in range(1, nbr):
        k = rng.integers(1, slots + 1) if br % 3 else slots - 1
        colind[br, :k] = np.sort(rng.choice(nbc, k, replace=False))
    return colind, slots


def test_blocked_ell_native_and_shim_against_the_closed_library(L, mode, capsys):
    """dense -> Blocked-ELL: b200dense2bell directly and the shim bit-identical to the closed convert, all on NaN-prefilled
    ellValue, with what the closed convert leaves in the -1 slots printed and asserted (zeros).  Blocked-ELL -> dense: refused by the
    closed library, so the shim forwards it unless switched on, and then matches the oracle and b200bell2dense"""
    cs, ours, closed = apis()
    rng = np.random.default_rng(41)
    pad_zero = []
    for m, n, bs in ((4, 6, 2), (64, 128, 16), (128, 96, 32)):
        for dt in (torch.float16, torch.float32, torch.float64):
            w = torch.empty(0, dtype=dt).element_size()
            colind, slots = bell_pattern(rng, m, n, bs)
            ci = dev(colind)
            padded = np.repeat(np.repeat(colind < 0, bs, axis=1), bs, axis=0).reshape(-1)     # elements of -1 slots in ellValue
            for order in (ROW, COL):
                ld = n if order == ROW else m
                src = torch.from_numpy(vals_bits(rng, m * n, w).reshape(-1)).cuda().view(dt)
                nan = lambda: torch.full((m * slots * bs * w,), 0xFF, dtype=torch.uint8, device="cuda").view(dt)  # noqa: E731
                want = cs.dense_to_sparse(closed, cs.CUSPARSE_FORMAT_BLOCKED_ELL, m, n, src, ld, order, colind=ci, ell_value=nan(),
                                          bs=bs).view(torch.uint8)
                wb = want.view(-1, w).cpu().numpy()
                pad_zero.append(bool((wb[padded] == 0).all()))
                assert pad_zero[-1], (m, bs, dt, order)
                ours.reset_stats()
                shim = cs.dense_to_sparse(ours, cs.CUSPARSE_FORMAT_BLOCKED_ELL, m, n, src, ld, order, colind=ci, ell_value=nan(), bs=bs)
                expect_counts(ours, route(L, 1, cs.CUSPARSE_FORMAT_BLOCKED_ELL, order, VTYPE[dt], m, n, m * slots * bs, bs))
                native = nan()
                assert L.b200dense2bell(stream(), m, n, bs, slots * bs, src.data_ptr(), ld, order, w, ci.data_ptr(), native.data_ptr(), 0) == 0
                torch.cuda.synchronize()
                case = (mode, m, n, bs, dt, order)
                assert torch.equal(native.view(torch.uint8), want), case
                assert torch.equal(shim.view(torch.uint8), want), case
                # Blocked-ELL -> dense
                ev = want.view(dt)
                dense = torch.full((ld * (m if order == ROW else n) * w,), 0x3C, dtype=torch.uint8, device="cuda").view(dt)
                ours.reset_stats()
                r = route(L, 0, cs.CUSPARSE_FORMAT_BLOCKED_ELL, order, VTYPE[dt], m, n, m * slots * bs, bs)
                try:
                    cs.sparse_to_dense(ours, cs.CUSPARSE_FORMAT_BLOCKED_ELL, m, n, ci, None, ev, dense, ld, order, bs=bs, ell_cols=slots * bs,
                                       query=not r)      # the closed bufferSize refuses Blocked-ELL; the native path needs no buffer
                    status = 0
                except cs.CuSparseError as e:
                    status = e.status
                assert status == (0 if r else cs.CUSPARSE_STATUS_NOT_SUPPORTED), status
                if r:
                    expect_counts(ours, 1)
                    oracle = R.bell_to_dense(np.full((ld * (m if order == ROW else n), w), 0x3C, np.uint8), m, n, ld, order, bs, colind,
                                             wb)
                    assert np.array_equal(dense.view(torch.uint8).cpu().numpy().reshape(-1, w), oracle), case
    with capsys.disabled():
        print(f"\nclosed dense->Blocked-ELL writes zeros into the -1 slots of NaN-prefilled ellValue: {all(pad_zero)} "
              f"({len(pad_zero)} cases)")


def test_the_routed_blocked_ell_class_runs_natively_and_bit_identically(L):
    """dense -> Blocked-ELL, row-major, bs 16, fp16 / fp32 at 8192^2: the class the route sends to b200dense2bell by default"""
    cs, ours, closed = apis()
    rng = np.random.default_rng(43)
    m = n = 8192
    bs = 16
    colind, slots = bell_pattern(rng, m, n, bs)
    ci = dev(colind)
    for dt in (torch.float16, torch.float32):
        w = torch.empty(0, dtype=dt).element_size()
        assert route(L, 1, cs.CUSPARSE_FORMAT_BLOCKED_ELL, ROW, VTYPE[dt], m, n, m * slots * bs, bs) == 1
        src = torch.randint(-1000, 1000, (m * n,), device="cuda").to(dt)
        res = []
        for api in (ours, closed):
            ev = torch.full((m * slots * bs * w,), 0xFF, dtype=torch.uint8, device="cuda").view(dt)
            ours.reset_stats()
            cs.dense_to_sparse(api, cs.CUSPARSE_FORMAT_BLOCKED_ELL, m, n, src, n, ROW, colind=ci, ell_value=ev, bs=bs)
            if api is ours:
                expect_counts(ours, 1)
            res.append(ev.view(torch.uint8))
        assert torch.equal(res[0], res[1]), dt


def sort_rows(off, ind, val):
    """each row's (index, value) pairs in ascending index order"""
    off, ind, val = off.cpu().numpy().astype(np.int64), ind.cpu().numpy(), val.view(torch.uint8).cpu().numpy().reshape(len(ind), -1)
    o = np.lexsort((ind, np.repeat(np.arange(len(off) - 1), np.diff(off - off[0]))))
    return ind[o], val[o]


def test_dense_to_csr_csc_through_the_shim_equals_the_closed_library(L, mode, capsys):
    """the closed convert orders columns within a row its own way: offsets bit for bit, each row's entries as a set (ours ascend)"""
    cs, ours, closed = apis()
    rng = np.random.default_rng(51)
    unsorted = 0
    for m, n in ((5, 4), (300, 257), (64, 4000)):
        for dt in (torch.float16, torch.bfloat16, torch.float32, torch.float64, torch.complex128):
            w = torch.empty(0, dtype=dt).element_size()
            for fmt in (cs.CUSPARSE_FORMAT_CSR, cs.CUSPARSE_FORMAT_CSC):
                for order in (ROW, COL):
                    for base in (0, 1):
                        ld = (n if order == ROW else m) + 1
                        bits = vals_bits(rng, ld * (m if order == ROW else n), w, zeros=True)
                        bits[rng.random(len(bits)) < 0.7] = 0
                        src = torch.from_numpy(bits.reshape(-1)).cuda().view(dt)
                        ours.reset_stats()
                        a = cs.dense_to_sparse(ours, fmt, m, n, src, ld, order, base)
                        s = ours.stats()
                        r = route(L, 1, fmt, order, VTYPE[dt], m, n, a[1].numel())
                        assert (s["native"], s["forwarded"]) == ((1, 0) if r else (0, 1)), s
                        b = cs.dense_to_sparse(closed, fmt, m, n, src, ld, order, base)
                        # the native entry point on the closed offsets
                        ind = torch.full_like(b[1], -7)
                        val = torch.full_like(b[2], float("nan"))
                        assert L.b200dense2csr(stream(), int(fmt == cs.CUSPARSE_FORMAT_CSC), m, n, b[1].numel(), src.data_ptr(), ld, order,
                                               VTYPE[dt], b[0].data_ptr(), ind.data_ptr(), val.data_ptr(), base) == 0
                        torch.cuda.synchronize()
                        assert torch.equal(a[0], b[0]), (m, n, dt, fmt, order, base)
                        si, sv = sort_rows(b[0], b[1], b[2])
                        if r:
                            assert np.array_equal(a[1].cpu().numpy(), si), (mode, m, n, dt, fmt, order, base)
                            assert np.array_equal(a[2].view(torch.uint8).cpu().numpy().reshape(len(si), -1), sv), (mode, m, n, dt, fmt)
                        else:
                            assert torch.equal(a[1], b[1]) and torch.equal(a[2].view(torch.uint8), b[2].view(torch.uint8))
                        unsorted += not np.array_equal(si, b[1].cpu().numpy())
                        assert np.array_equal(ind.cpu().numpy(), si), (m, n, dt, fmt, order, base)
                        assert np.array_equal(val.view(torch.uint8).cpu().numpy().reshape(len(si), -1), sv), (m, n, dt, fmt, order, base)
    with capsys.disabled():
        print(f"\nclosed DenseToSparse_convert left the indices of a row unsorted in {unsorted} of 120 cases")


def pinned_values():
    """the predicate fixture: signed zeros, denormals, NaN / Inf, complex values with one zero part"""
    f32 = np.array([0.0, -0.0, 1e-45, -1e-45, 1e-40, np.nan, np.inf, -np.inf, 1.0, 0.0], np.float32)
    f64 = np.array([0.0, -0.0, 5e-324, -5e-324, 1e-310, np.nan, np.inf, -np.inf, 1.0, 0.0], np.float64)
    f16 = np.array([0.0, -0.0, 6e-8, -6e-8, 3e-5, np.nan, np.inf, -np.inf, 1.0, 0.0], np.float16)
    bf16 = np.array([0x0000, 0x8000, 0x0001, 0x8001, 0x0040, 0x7FC1, 0x7F80, 0xFF80, 0x3F80, 0x0000], np.uint16)
    c128 = np.array([0, -0.0 + 0j, 1j * 5e-324, complex(-0.0, -0.0), complex(0, -0.0), complex(np.nan, 0), complex(0, np.inf), 1 + 0j,
                     complex(0.0, 1.0), 0], np.complex128)
    c64 = np.array([0, -0.0 + 0j, 1j * 1e-45, complex(-0.0, -0.0), complex(0, -0.0), complex(np.nan, 0), complex(0, np.inf), 1 + 0j,
                    complex(0.0, 1.0), 0], np.complex64)
    return {torch.float32: f32, torch.float64: f64, torch.float16: f16, torch.bfloat16: bf16, torch.complex64: c64,
            torch.complex128: c128}


def test_zero_predicate_matches_the_closed_analysis(L, capsys):
    cs, ours, closed = apis()
    for dt, arr in pinned_values().items():
        w = torch.empty(0, dtype=dt).element_size()
        src = torch.from_numpy(arr.copy()).cuda().view(dt).reshape(1, -1).repeat(3, 1).reshape(-1)
        got = {}
        for name, api in (("ours", ours), ("closed", closed)):
            got[name] = cs.dense_to_sparse(api, cs.CUSPARSE_FORMAT_CSR, 3, len(arr), src, len(arr), ROW)
        kept = sorted(got["closed"][1][:len(got["closed"][1]) // 3].tolist())
        with capsys.disabled():
            print(f"\nclosed dense->CSR keeps {dt} positions {kept} of {arr.tolist()}")
        mine = np.nonzero(R.nonzero(arr.view(np.uint8).reshape(len(arr), w), w // 2 if dt.is_complex else w))[0].tolist()
        assert kept == mine, (dt, kept, mine)
        off = got["closed"][0]
        ind = torch.full_like(got["closed"][1], -7)
        val = torch.full_like(got["closed"][2], 0)
        assert L.b200dense2csr(stream(), 0, 3, len(arr), ind.numel(), src.data_ptr(), len(arr), ROW, VTYPE[dt], off.data_ptr(),
                               ind.data_ptr(), val.data_ptr(), 0) == 0
        torch.cuda.synchronize()
        si, sv = sort_rows(off, got["closed"][1], got["closed"][2])
        assert np.array_equal(ind.cpu().numpy(), si) and np.array_equal(val.view(torch.uint8).cpu().numpy().reshape(len(si), -1), sv), dt
        assert torch.equal(got["ours"][0], off)


@pytest.mark.parametrize("dt", [torch.float16, torch.bfloat16])
def test_zero_predicate_over_every_16_bit_pattern(L, dt):
    """all 65536 bit patterns in one row: the closed analysis' kept set, the oracle's and the native convert's agree"""
    cs, _, closed = apis()
    bits = np.arange(65536, dtype=np.uint32).astype(np.uint16)
    src = torch.from_numpy(bits.view(np.int16).copy()).cuda().view(dt)
    off, ind, val = cs.dense_to_sparse(closed, cs.CUSPARSE_FORMAT_CSR, 1, 65536, src, 65536, ROW)
    kept = np.zeros(65536, bool)
    kept[ind.cpu().numpy()] = True
    assert np.array_equal(kept, R.nonzero(bits.view(np.uint8).reshape(-1, 2), 2))
    mine = torch.full_like(ind, -7)
    assert L.b200dense2csr(stream(), 0, 1, 65536, ind.numel(), src.data_ptr(), 65536, ROW, VTYPE[dt], off.data_ptr(), mine.data_ptr(),
                           torch.empty_like(val).data_ptr(), 0) == 0
    torch.cuda.synchronize()
    assert np.array_equal(mine.cpu().numpy(), np.nonzero(kept)[0])


def test_duplicates_in_sparse_to_dense(L, capsys):
    """CSR rows with repeated columns (in one 32-entry chunk and across chunks): the last in storage order wins in ours; the
    closed library's behaviour is printed and compared"""
    cs, ours, closed = apis()
    rng = np.random.default_rng(61)
    m, n = 64, 128                                   # 56 entries per row, repeats within a 32-entry chunk and across chunks
    cols = [np.concatenate([rng.choice(n, 16, replace=False), rng.integers(0, n, 40)]) for _ in range(m)]
    off = np.concatenate([[0], np.cumsum([len(c) for c in cols])])
    ind = np.concatenate(cols)
    vals = torch.arange(1, len(ind) + 1, dtype=torch.float32, device="cuda")
    dense = torch.zeros(m * n, dtype=torch.float32, device="cuda")
    cs.sparse_to_dense(closed, cs.CUSPARSE_FORMAT_CSR, m, n, dev(off), dev(ind), vals, dense, n, ROW)
    mine = torch.full((m * n,), 7.0, dtype=torch.float32, device="cuda")
    assert L.b200csr2dense(stream(), 0, m, n, len(ind), dev(off).data_ptr(), dev(ind).data_ptr(), vals.data_ptr(), 4, 0, mine.data_ptr(), n,
                           ROW) == 0
    torch.cuda.synchronize()
    closed_res = dense.cpu().numpy()
    v = vals.cpu().numpy().view(np.uint8).reshape(-1, 4)
    last = R.csr_to_dense(np.zeros((m * n, 4), np.uint8), m, n, n, ROW, off, ind, v).reshape(-1).view(np.float32)
    rows = np.repeat(np.arange(m), np.diff(off))
    first = R.scatter(np.zeros((m * n, 4), np.uint8), m, n, n, ROW, rows[::-1], ind[::-1], v[::-1]).reshape(-1).view(np.float32)
    total = np.zeros(m * n, np.float64)
    np.add.at(total, rows * n + ind, vals.cpu().numpy())
    verdict = ("last wins" if np.array_equal(closed_res, last) else "first wins" if np.array_equal(closed_res, first)
               else "summed" if np.allclose(closed_res, total) else "one of them, in no storage order" if
               np.isin(closed_res[total != 0], vals.cpu().numpy()).all() else "other")
    with capsys.disabled():
        print(f"\nclosed SparseToDense with duplicate CSR entries: {verdict}")
    assert np.array_equal(mine.cpu().numpy(), last)
    if route(L, 0, cs.CUSPARSE_FORMAT_CSR, ROW, 0, m, n, len(ind)):
        assert verdict == "last wins"


def test_nnz_refresh_lets_spmv_and_spmm_run_on_a_converted_matrix(L):
    """dense -> CSR through analysis / cusparseCsrSetPointers / convert, then cusparseSpMV and cusparseSpMM through the shim on
    that descriptor: the side table must hold the nnz the analysis set, not the 0 of cusparseCreateCsr"""
    import scipy.sparse as sp
    cs, ours, _ = apis()
    rng = np.random.default_rng(71)
    m, n, k = 500, 300, 8
    A = np.where(rng.random((m, n)) < 0.05, rng.standard_normal((m, n)), 0.0)
    x = rng.standard_normal(n)
    X = rng.standard_normal((n, k))
    src = torch.from_numpy(A.reshape(-1).copy()).cuda()
    got = {}

    def then(h, matB):
        xd, yd = torch.from_numpy(x).cuda(), torch.zeros(m, dtype=torch.float64, device="cuda")
        vx, vy = ours.cusparseCreateDnVec(n, xd), ours.cusparseCreateDnVec(m, yd)
        alpha, beta = C.c_double(1.0), C.c_double(0.0)
        size = C.c_size_t()
        ours._call(ours.lib, "cusparseSpMV_bufferSize", h, 0, C.byref(alpha), matB, vx, C.byref(beta), vy, 1, 0, C.byref(size))
        buf = torch.empty(max(size.value, 16), dtype=torch.uint8, device="cuda")
        ours._call(ours.lib, "cusparseSpMV", h, 0, C.byref(alpha), matB, vx, C.byref(beta), vy, 1, 0, cs._ptr(buf))
        Xd, Yd = torch.from_numpy(X.T.copy().reshape(-1)).cuda(), torch.zeros(m * k, dtype=torch.float64, device="cuda")
        mb, mc = ours.cusparseCreateDnMat(n, k, n, Xd), ours.cusparseCreateDnMat(m, k, m, Yd)
        ours._call(ours.lib, "cusparseSpMM_bufferSize", h, 0, 0, C.byref(alpha), matB, mb, C.byref(beta), mc, 1, 0, C.byref(size))
        buf2 = torch.empty(max(size.value, 16), dtype=torch.uint8, device="cuda")
        ours._call(ours.lib, "cusparseSpMM", h, 0, 0, C.byref(alpha), matB, mb, C.byref(beta), mc, 1, 0, cs._ptr(buf2))
        torch.cuda.synchronize()
        got["y"], got["Y"] = yd.cpu().numpy(), Yd.cpu().numpy().reshape(k, m).T
        ours.cusparseDestroyDnVec(vx), ours.cusparseDestroyDnVec(vy), ours.cusparseDestroyDnMat(mb), ours.cusparseDestroyDnMat(mc)

    cs.dense_to_sparse(ours, cs.CUSPARSE_FORMAT_CSR, m, n, src, n, ROW, then=then)
    S = sp.csr_matrix(A)
    assert np.allclose(got["y"], S @ x, rtol=1e-12, atol=1e-12)
    assert np.allclose(got["Y"], S @ X, rtol=1e-12, atol=1e-12)


def test_reference_samples_pass_on_the_shim(L):
    for s, call in (("sparse2dense_csr", "SparseToDense"), ("dense2sparse_csr", "DenseToSparse_convert"),
                    ("dense2sparse_blockedell", "DenseToSparse_convert")):
        exe = os.path.join(ROOT, "oracle", "_ref", f"{s}_example.b200")
        if not os.path.exists(exe):
            pytest.skip("oracle/_ref not built (needs the reference checkout at build time)")
        for suffix in ("cusparse", "b200"):
            p = subprocess.run([exe[:-4] + suffix], capture_output=True, text=True, env=dict(os.environ, B200SPMV_LOG="1"), timeout=300)
            assert p.returncode == 0 and "PASSED" in p.stdout, (s, suffix, p.stdout + p.stderr)
        print(s, re.findall(r"\[b200spmv\] " + call + r" (native|forwarded)", p.stderr))
