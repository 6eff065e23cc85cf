"""GPU: the native routes at the largest sizes they admit, and one past where that is cheap, checked BIT FOR BIT against the int64
reference of oracle/limits.py (integer data: every partial sum below 2^24, so fp32, fp64 and every summation order give the same
value).  The data is built on the device from closed-form index formulas; every index extreme carries a non-zero (column 0, the
last column, 2^31 - 1 and 2^31 where they exist, the first and the last row, an empty row, rows that cross tiles).

  A. launch caps: CSR SpMM (b200spmm_csr_ws, cusparseSpMM, b200spmm_csr_t, b200spmm_csr16) at N = 32 * 65535 (the last N whose
     transpose of a column-major B fits one grid.y), one past it and 64 * 65535 - 1 (the largest N admitted; 32 * 65535 for 16-bit
     values); COO SpMM and CSR SDDMM one past the transpose's former cap and at COO's panel cap; strided batches of 65535 (CSR
     SDDMM, COO SpMM, BSR SpMM, BSR SDDMM).
  B. 32-bit counts: CSR SpMV at the largest nnz the specialised kernels take (INT32_MAX - 65537) on the flat, tile, short and
     transpose kernels, one past it on csr_generic_kernel; COO SpMV (tile, seg) and Sliced-ELL SpMV (slice 32, 7) at that nnz;
     rows at INT32_MAX - 65 (short kernel) and in the band above it (csr_generic_kernel).
  C. 64-bit values: b200spmv_csr_generic_mv with columns past 2^31 and with row offsets past 2^31, b200spmv_sell_generic_mv with
     slice offsets past 2^31, b200spmv_coo_generic_mv with row indices past 2^31.

Each case states its footprint in GB from the element counts and the plan sizes (host functions) and skips, with the numbers, when
the device has less free memory; everything is freed at the end of a case.  Peaks (torch.cuda.max_memory_allocated) are printed
per case with -s."""
import ctypes as C
import gc

import pytest
import torch

from oracle import limits as LM

pytestmark = pytest.mark.gpu

M = LM.INT32_MAX
NNZ_FAST = M - 65537
BIG = 2**31 + 2**20
COLS_B = 1 << 21                    # columns of the group B matrices: fan-in ~1K spread + 32K on the hot columns
TD = {0: torch.float32, 1: torch.float64}


@pytest.fixture(scope="module")
def N():
    if not torch.cuda.is_available():
        pytest.skip("no GPU")
    from cudalibrarysamples_b200 import build, lib
    lib.shim()
    return lib.load(build.LIB_PATH)


@pytest.fixture(scope="module")
def cs():
    from cudalibrarysamples_b200 import cusparse_api
    return cusparse_api


@pytest.fixture(scope="module")
def api(cs, N):
    a = cs.Api("b200")
    a.set_option("B200SPMV_GENERIC", "csr")
    return a


def stream():
    return torch.cuda.current_stream().cuda_stream


def guard(name, need_bytes):
    """skip when the device has less free memory than the case needs (plus 1 GB for torch and the library)"""
    torch.cuda.synchronize()
    gc.collect()
    torch.cuda.empty_cache()
    free, total = torch.cuda.mem_get_info()
    need = need_bytes + (1 << 30)
    if free < need:
        pytest.skip(f"{name}: needs {LM.gb(need):.1f} GB, {LM.gb(free):.1f} of {LM.gb(total):.1f} GB free")
    torch.cuda.reset_peak_memory_stats()


def release(name):
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated()
    gc.collect()
    torch.cuda.empty_cache()
    print(f"\n[limits] {name}: peak {LM.gb(peak):.2f} GB allocated")


def scal(v, dt):
    c = (C.c_double if dt == 1 else C.c_float)(v)
    return C.cast(C.pointer(c), C.c_void_p), c


def as_dt(t_int64, dt):
    return t_int64.to(TD[dt])


def exact(got, want_int64):
    """bit equality of a float result with the int64 reference (both hold small integers, so the float conversion is exact)"""
    assert not torch.isnan(got).any(), "an output element was never written"
    assert torch.equal(got.to(torch.float64), want_int64.to(torch.float64))


# =============================================================================================================== A. launch caps
A_ROWS, A_COLS = 8, 3
A_OFF = [0, 2, 3, 3, 5, 6, 8, 9, 11]     # row 2 empty, rows 0 and 7 stored
N_CAPS = [32 * 65535, 32 * 65535 + 1, 64 * 65535 - 1]


def a_matrix(base):
    off = torch.tensor(A_OFF, dtype=torch.int64, device="cuda")
    nnz = A_OFF[-1]
    col = LM.fill(torch.empty(nnz, dtype=torch.int64, device="cuda"), lambda k: (k * 2) % A_COLS)
    col[0] = 0
    col[-1] = A_COLS - 1
    val = LM.fill(torch.empty(nnz, dtype=torch.int64, device="cuda"), LM.val_at)
    return off, col, val


def dense(rows, n, row_major, seed):
    """an int64 rows x n matrix of small non-zeros and its storage (1-D, tight leading dimension) in the given order"""
    i = torch.arange(rows * n, dtype=torch.int64, device="cuda").view(rows, n)
    m = LM.small(i * 7 + seed)
    return m, (m if row_major else m.t()).reshape(-1)


def spmm_ref(off, col, val, B, transpose=False):
    """int64 alpha * op(A) B, A tiny (loop over its entries)"""
    rows = off.numel() - 1
    out = torch.zeros(((A_COLS if transpose else rows), B.shape[1]), dtype=torch.int64, device="cuda")
    offl, coll, vall = off.tolist(), col.tolist(), val.tolist()
    for r in range(rows):
        for p in range(offl[r], offl[r + 1]):
            if transpose:
                out[coll[p]] += vall[p] * B[r]
            else:
                out[r] += vall[p] * B[coll[p]]
    return LM.ALPHA * out


def c_view(buf, rows, n, row_major):
    return buf.view(rows, n) if row_major else buf.view(n, rows).t()


@pytest.mark.parametrize("n", N_CAPS)
@pytest.mark.parametrize("dt", [0, 1])
def test_spmm_csr_at_the_n_caps(N, api, cs, n, dt):
    """b200spmm_csr_ws and cusparseSpMM (CSR, opA = N), B and C in both orders, base 0 and 1; beta = 0 into a NaN C and beta = 3"""
    vsz = 8 if dt else 4
    ws = N.b200spmm_csr_workspace_bytes(dt, A_COLS, n, 0)
    need = (A_COLS * n + 3 * A_ROWS * n) * vsz + ws + 3 * A_ROWS * n * 8
    guard(f"spmm csr n={n}", need)
    torch.cuda.synchronize()
    for base in (0, 1):
        off, col, val = a_matrix(0)
        offd, cold, vald = (off + base).int(), (col + base).int(), as_dt(val, dt)
        Bm, _ = dense(A_COLS, n, True, 1)
        want = spmm_ref(off, col, val, Bm)
        wsb = torch.empty(max(ws, 16), dtype=torch.uint8, device="cuda")
        for b_row in (0, 1):
            Bs = as_dt((Bm if b_row else Bm.t()).reshape(-1), dt)
            for c_row in (0, 1):
                for beta in (0, LM.BETA):
                    y0m, y0s = dense(A_ROWS, n, c_row, 2)
                    Cb = torch.full((A_ROWS * n,), float("nan"), dtype=TD[dt], device="cuda") if beta == 0 else as_dt(y0s, dt)
                    pa, _ka = scal(LM.ALPHA, dt)
                    pb, _kb = scal(beta, dt)
                    rc = N.b200spmm_csr_ws(stream(), dt, A_ROWS, A_COLS, n, off[-1].item(), offd.data_ptr(), cold.data_ptr(),
                                           vald.data_ptr(), base, pa, pb, 0, Bs.data_ptr(), n if b_row else A_COLS, b_row,
                                           Cb.data_ptr(), n if c_row else A_ROWS, c_row, wsb.data_ptr())
                    torch.cuda.synchronize()
                    assert rc == 0, (base, b_row, c_row, beta, rc)
                    exact(c_view(Cb, A_ROWS, n, c_row), want + (LM.BETA * y0m if beta else 0))
                    del Cb
                # the same call through the shim: served natively
                y0m, y0s = dense(A_ROWS, n, c_row, 2)
                api.reset_stats()
                Cs = cs.spmm(api, A_ROWS, A_COLS, dict(off=offd, col=cold, val=vald), Bs, as_dt(y0s, dt), alpha=LM.ALPHA,
                             beta=LM.BETA, order_b=cs.CUSPARSE_ORDER_ROW if b_row else cs.CUSPARSE_ORDER_COL,
                             order_c=cs.CUSPARSE_ORDER_ROW if c_row else cs.CUSPARSE_ORDER_COL, base=base, n=n)
                st = api.stats()
                assert (st["native"], st["forwarded"]) == (1, 0), st
                exact(c_view(Cs, A_ROWS, n, c_row), want + LM.BETA * y0m)
                del Cs
            del Bs
    release(f"spmm csr n={n} dt={dt}")


F16, BF16 = 2, 14
TD16 = {F16: torch.float16, BF16: torch.bfloat16}


@pytest.mark.parametrize("dt,n", [(0, N_CAPS[1]), (0, N_CAPS[2]), (1, N_CAPS[1]), (1, N_CAPS[2]), (F16, 32 * 65535), (BF16, 32 * 65535)])
def test_spmm_csr_t_at_the_n_caps(N, n, dt):
    """b200spmm_csr_t (A^T B through the opA = N kernels on the transposed plan), column-major B and C, base 0 and 1: fp32 / fp64 past
    32 * 65535 up to 64 * 65535 - 1, fp16 / bf16 (into an fp32 C) at their cap 32 * 65535.  cusparseSpMM with opA = T forwards these
    shapes (its native class is N <= 256, DESIGN.md 3.22), so the entry point is called directly."""
    h16 = dt in TD16
    ct = 0 if h16 else dt
    vsz = 2 if h16 else (8 if dt else 4)
    sbk, sbj = 1, A_ROWS                                  # op(B) = B: A_ROWS x n, column-major
    ws = N.b200spmm_csr_t_workspace_bytes(dt, A_ROWS, A_COLS, n, A_OFF[-1], sbk, sbj)
    assert ws > 0
    guard(f"spmm csr_t n={n}", (A_ROWS * n + 2 * A_COLS * n) * vsz + ws + 2 * A_COLS * n * 8 + A_ROWS * n * 8)
    for base in (0, 1):
        off, col, val = a_matrix(0)
        Bm, _ = dense(A_ROWS, n, True, 3)
        want = spmm_ref(off, col, val, Bm, transpose=True)
        Bs = (Bm.t().reshape(-1).to(TD16[dt])) if h16 else as_dt(Bm.t().reshape(-1), dt)
        Cb = torch.full((A_COLS * n,), float("nan"), dtype=TD[ct], device="cuda")
        wsb = torch.empty(ws, dtype=torch.uint8, device="cuda")
        pa, _ka = scal(LM.ALPHA, ct)
        pb, _kb = scal(0, ct)
        offd, cold = (off + base).int(), (col + base).int()           # named: alive until the kernels ran
        vald = val.to(TD16[dt]) if h16 else as_dt(val, dt)
        rc = N.b200spmm_csr_t(stream(), dt, ct, A_ROWS, A_COLS, n, A_OFF[-1], offd.data_ptr(), cold.data_ptr(), vald.data_ptr(), base,
                              pa, pb, 0, Bs.data_ptr(), sbk, sbj, Cb.data_ptr(), A_COLS, 0, 0, wsb.data_ptr(), ws)
        torch.cuda.synchronize()
        assert rc == 0, rc
        exact(c_view(Cb, A_COLS, n, 0), want)
        del Bs, Cb, wsb
    release(f"spmm csr_t n={n} dt={dt}")


@pytest.mark.parametrize("dt", [F16, BF16])
def test_spmm_csr16_at_its_n_cap(N, dt):
    """b200spmm_csr16 (opA = N) at N = 32 * 65535, its cap: column-major B (copied row-major in the workspace) into an fp32 C in both
    orders, base 0 and 1.  cusparseSpMM forwards 16-bit CSR at this N (its native class is N <= 256, DESIGN.md 3.18)."""
    n = 32 * 65535
    sbk, sbj = 1, A_COLS
    ws = N.b200spmm_csr16_workspace_bytes(A_COLS, n, A_OFF[-1], sbk, sbj)
    guard(f"spmm csr16 n={n}", A_COLS * n * 2 + A_ROWS * n * 4 + ws + 3 * A_ROWS * n * 8)
    pa, _ka = scal(LM.ALPHA, 0)
    pb, _kb = scal(0, 0)
    for base in (0, 1):
        off, col, val = a_matrix(0)
        Bm, _ = dense(A_COLS, n, True, 1)
        want = spmm_ref(off, col, val, Bm)
        Bs = Bm.t().reshape(-1).to(TD16[dt])
        offd, cold, vald = (off + base).int(), (col + base).int(), val.to(TD16[dt])
        wsb = torch.empty(max(ws, 16), dtype=torch.uint8, device="cuda")
        for c_row in (0, 1):
            Cb = torch.full((A_ROWS * n,), float("nan"), dtype=torch.float32, device="cuda")
            rc = N.b200spmm_csr16(stream(), dt, 0, A_ROWS, A_COLS, n, A_OFF[-1], offd.data_ptr(), cold.data_ptr(), vald.data_ptr(), base,
                                  pa, pb, 0, Bs.data_ptr(), sbk, sbj, Cb.data_ptr(), n if c_row else A_ROWS, c_row, wsb.data_ptr(), ws)
            torch.cuda.synchronize()
            assert rc == 0, rc
            exact(c_view(Cb, A_ROWS, n, c_row), want)
            del Cb
        del Bs, wsb
    release(f"spmm csr16 dt={dt}")


@pytest.mark.parametrize("n", N_CAPS[1:], ids=["past_transpose_cap", "panel_cap"])
@pytest.mark.parametrize("dt", [0, 1])
def test_spmm_coo_and_sddmm_past_the_former_transpose_cap(N, dt, n):
    """b200spmm_coo and b200sddmm_csr copy a column-major operand row-major through spmm_transpose_b_kernel at N = K =
    32 * 65535 + 1 (they used to fall back to strided reads there) and at 64 * 65535 - 1 (COO SpMM's panel cap, (N + 63) / 64 <=
    65535); beta = 0 into NaN"""
    vsz = 8 if dt else 4
    off, col, val = a_matrix(0)
    nnz = A_OFF[-1]
    row = torch.searchsorted(off, torch.arange(nnz, device="cuda"), right=True) - 1
    ws = N.b200spmm_coo_workspace_bytes(dt, 0, A_ROWS, A_COLS, n, nnz, 0, 1, 0)
    wsd = N.b200sddmm_csr_workspace_bytes(dt, A_ROWS, A_COLS, n, 1, A_ROWS, A_COLS, 1, 1, 0, 0)
    assert ws >= A_COLS * n * vsz and wsd >= (A_ROWS + A_COLS) * n * vsz
    guard(f"coo / sddmm n={n}", (A_COLS * n + 2 * A_ROWS * n) * vsz + max(ws, wsd) + 4 * A_ROWS * n * 8)
    pa, _ka = scal(LM.ALPHA, dt)
    pb, _kb = scal(0, dt)
    for base in (0, 1):
        # COO SpMM, B and C column-major
        Bm, _ = dense(A_COLS, n, True, 1)
        Bs = as_dt(Bm.t().reshape(-1), dt)
        Cb = torch.full((A_ROWS * n,), float("nan"), dtype=TD[dt], device="cuda")
        wsb = torch.empty(ws, dtype=torch.uint8, device="cuda")
        rowd, offd, cold, vald = (row + base).int(), (off + base).int(), (col + base).int(), as_dt(val, dt)
        rc = N.b200spmm_coo(stream(), dt, 0, A_ROWS, A_COLS, n, nnz, rowd.data_ptr(), cold.data_ptr(), vald.data_ptr(), base, pa, pb, 0,
                            Bs.data_ptr(), A_COLS, 0, Cb.data_ptr(), A_ROWS, 0, 1, 0, 0, 0, wsb.data_ptr(), ws)
        torch.cuda.synchronize()
        assert rc == 0, rc
        exact(c_view(Cb, A_ROWS, n, 0), spmm_ref(off, col, val, Bm))
        del Bs, Cb, wsb
        # CSR SDDMM: C = alpha * (A B) o spy(C), A (A_ROWS x K) and B (K x A_COLS) both stored the K-strided way round
        Am = LM.small(torch.arange(A_ROWS * n, dtype=torch.int64, device="cuda").view(A_ROWS, n) + 4)
        # B non-zero on every 8th k only (the last k, 32 * 65535, among them): K-sums stay below 2^24
        kk = torch.arange(n * A_COLS, dtype=torch.int64, device="cuda").view(n, A_COLS)
        Bk = torch.where((kk // A_COLS) % 8 == 0, LM.small(kk * 5 + 1), 0)
        del kk
        As, Bks = as_dt(Am.t().reshape(-1), dt), as_dt(Bk.reshape(-1), dt)       # A column-major (sak = A_ROWS), B row-major (sbk = A_COLS)
        vals = torch.full((nnz,), float("nan"), dtype=TD[dt], device="cuda")
        wsb = torch.empty(wsd, dtype=torch.uint8, device="cuda")
        rc = N.b200sddmm_csr(stream(), dt, A_ROWS, A_COLS, n, nnz, offd.data_ptr(), cold.data_ptr(), vals.data_ptr(), base, pa, pb, 0,
                             As.data_ptr(), 1, A_ROWS, Bks.data_ptr(), A_COLS, 1, 1, 0, 0, 0, 0, wsb.data_ptr(), wsd)
        torch.cuda.synchronize()
        assert rc == 0, rc
        want = torch.stack([(Am[r] * Bk[:, c]).sum() for r, c in zip(row.tolist(), col.tolist())]) * LM.ALPHA
        exact(vals, want)
        del As, Bks, vals, wsb, Am, Bk
    release(f"coo / sddmm n={n} dt={dt}")


BATCH = 65535
K_B, N_B = 4, 4                       # the inner and the dense dimension of the batched products
B_OFF, B_COL, BS = [0, 2, 2, 3], [0, 1, 1], 2      # BSR: 3 block-rows (the middle one empty) x 2 block-columns, 2 x 2 blocks


def batched(shape, seed):
    """an int64 (BATCH, *shape) tensor of small non-zeros, different in every matrix of the batch"""
    n = 1
    for d in shape:
        n *= d
    return LM.small(torch.arange(BATCH * n, dtype=torch.int64, device="cuda").view(BATCH, *shape) * 5 + seed)


def bsr_dense(vals):
    """(BATCH, 6, 4) dense matrices of the BSR pattern holding vals (BATCH, 3, BS, BS), blocks row-major"""
    d = torch.zeros(BATCH, 3 * BS, 2 * BS, dtype=torch.int64, device="cuda")
    brow = [r for r in range(3) for _ in range(B_OFF[r], B_OFF[r + 1])]
    for p, (br, bc) in enumerate(zip(brow, B_COL)):
        d[:, br * BS:(br + 1) * BS, bc * BS:(bc + 1) * BS] = vals[:, p]
    return d


def bmm(a, b):
    """exact int64 batched product of small integers (through fp64: every sum stays far below 2^53)"""
    return torch.bmm(a.double(), b.double()).round().long()


@pytest.mark.parametrize("dt", [0, 1])
def test_strided_batches_at_65535(N, dt):
    """batch = 65535, the largest the batched entry points take (grid.y / grid.z), on tiny matrices: CSR SDDMM, COO SpMM, BSR SpMM and
    BSR SDDMM, every operand strided (the sparsity pattern shared), beta = 0 into NaN.  Each matrix of the batch holds other values,
    so a batch index that wraps or stops early shows."""
    guard("strided batches", 64 << 20)
    pa, _ka = scal(LM.ALPHA, dt)
    pb, _kb = scal(0, dt)
    off, col, _ = a_matrix(0)
    nnz = A_OFF[-1]
    row = torch.searchsorted(off, torch.arange(nnz, device="cuda"), right=True) - 1
    offd, cold = off.int(), col.int()
    # CSR SDDMM: C_b = alpha * (A_b B_b) o spy(C), A_b 8 x K row-major, B_b K x 3 row-major; columns / values strided by nnz
    A, B = batched((A_ROWS, K_B), 1), batched((K_B, A_COLS), 2)
    Ad, Bd = as_dt(A.reshape(-1), dt), as_dt(B.reshape(-1), dt)
    colt = cold.repeat(BATCH)
    vals = torch.full((BATCH * nnz,), float("nan"), dtype=TD[dt], device="cuda")
    wsd = N.b200sddmm_csr_workspace_bytes(dt, A_ROWS, A_COLS, K_B, K_B, 1, A_COLS, 1, BATCH, A_ROWS * K_B, K_B * A_COLS)
    wsb = torch.empty(max(wsd, 16), dtype=torch.uint8, device="cuda")
    rc = N.b200sddmm_csr(stream(), dt, A_ROWS, A_COLS, K_B, nnz, offd.data_ptr(), colt.data_ptr(), vals.data_ptr(), 0, pa, pb, 0,
                         Ad.data_ptr(), K_B, 1, Bd.data_ptr(), A_COLS, 1, BATCH, 0, nnz, A_ROWS * K_B, K_B * A_COLS, wsb.data_ptr(), wsd)
    torch.cuda.synchronize()
    assert rc == 0, rc
    exact(vals.view(BATCH, nnz), LM.ALPHA * bmm(A, B)[:, row, col])
    del vals, colt, wsb
    # COO SpMM: C_b = alpha * A_b B_b, A_b 8 x 3 with the values of matrix b, B_b 3 x N_B and C_b column-major
    V = batched((nnz,), 3)
    Adense = torch.zeros(BATCH, A_ROWS, A_COLS, dtype=torch.int64, device="cuda")
    Adense[:, row, col] = V
    Bc = batched((A_COLS, N_B), 4)
    rowt, colt, valt = row.int().repeat(BATCH), cold.repeat(BATCH), as_dt(V.reshape(-1), dt)
    Bs = as_dt(Bc.transpose(1, 2).reshape(-1), dt)
    Cb = torch.full((BATCH * A_ROWS * N_B,), float("nan"), dtype=TD[dt], device="cuda")
    ws = N.b200spmm_coo_workspace_bytes(dt, 0, A_ROWS, A_COLS, N_B, nnz, 0, BATCH, A_COLS * N_B)
    wsb = torch.empty(max(ws, 16), dtype=torch.uint8, device="cuda")
    rc = N.b200spmm_coo(stream(), dt, 0, A_ROWS, A_COLS, N_B, nnz, rowt.data_ptr(), colt.data_ptr(), valt.data_ptr(), 0, pa, pb, 0,
                        Bs.data_ptr(), A_COLS, 0, Cb.data_ptr(), A_ROWS, 0, BATCH, nnz, A_COLS * N_B, A_ROWS * N_B, wsb.data_ptr(), ws)
    torch.cuda.synchronize()
    assert rc == 0, rc
    exact(Cb.view(BATCH, N_B, A_ROWS).transpose(1, 2), LM.ALPHA * bmm(Adense, Bc))
    del rowt, colt, valt, Bs, Cb, wsb
    # BSR SpMM: C_b (6 x N_B, row-major) = alpha * A_b B_b, A_b's blocks strided, B_b 4 x N_B row-major
    bnnz, m, k = B_OFF[-1], 3 * BS, 2 * BS
    BV = batched((bnnz, BS, BS), 5)
    boff, bcol = torch.tensor(B_OFF, dtype=torch.int32, device="cuda"), torch.tensor(B_COL, dtype=torch.int32, device="cuda")
    bv, Bb = as_dt(BV.reshape(-1), dt), batched((k, N_B), 6)
    Bbs = as_dt(Bb.reshape(-1), dt)
    Cb = torch.full((BATCH * m * N_B,), float("nan"), dtype=TD[dt], device="cuda")
    ws = N.b200spmm_bsr_workspace_bytes(dt, m, N_B, BS, bnnz, BATCH)
    wsb = torch.empty(max(ws, 16), dtype=torch.uint8, device="cuda")
    rc = N.b200spmm_bsr(stream(), dt, dt, m, k, N_B, BS, bnnz, boff.data_ptr(), bcol.data_ptr(), bv.data_ptr(), 0, 1, pa, pb, 0,
                        Bbs.data_ptr(), N_B, 1, Cb.data_ptr(), N_B, 1, BATCH, 0, 0, bnnz * BS * BS, k * N_B, m * N_B, wsb.data_ptr(), ws)
    torch.cuda.synchronize()
    assert rc == 0, rc
    exact(Cb.view(BATCH, m, N_B), LM.ALPHA * bmm(bsr_dense(BV), Bb))
    del bv, Bbs, Cb, wsb
    # BSR SDDMM: the blocks of C_b (6 x 4) = alpha * (A_b B_b) on the pattern, A_b 6 x K_B and B_b K_B x 4 row-major
    Aq, Bq = batched((m, K_B), 7), batched((K_B, k), 8)
    Aqs, Bqs = as_dt(Aq.reshape(-1), dt), as_dt(Bq.reshape(-1), dt)
    cv = torch.full((BATCH * bnnz * BS * BS,), float("nan"), dtype=TD[dt], device="cuda")
    rc = N.b200sddmm_bsr(stream(), dt, dt, m, k, K_B, BS, bnnz, boff.data_ptr(), bcol.data_ptr(), cv.data_ptr(), 0, 1, pa, pb, 0,
                         Aqs.data_ptr(), K_B, 1, Bqs.data_ptr(), k, 1, BATCH, 0, 0, bnnz * BS * BS, m * K_B, K_B * k)
    torch.cuda.synchronize()
    assert rc == 0, rc
    P = LM.ALPHA * bmm(Aq, Bq)
    brow = [r for r in range(3) for _ in range(B_OFF[r], B_OFF[r + 1])]
    want = torch.stack([P[:, br * BS:(br + 1) * BS, bc * BS:(bc + 1) * BS] for br, bc in zip(brow, B_COL)], dim=1)
    exact(cv.view(BATCH, bnnz, BS, BS), want)


@pytest.mark.parametrize("dt", [0, 1])
def test_strided_batch_csr_spmm_at_65535(N, cs, api, dt):
    """cusparseSpMM on a CSR A with a strided batch of 65535 tiny products (B200SPMV_GENERIC=all: the shim's loop of one
    b200spmm_csr_ws per matrix): A_b's columns and values strided, offsets shared, B_b column-major (copied row-major in the buffer
    by every product), C_b column-major, beta = 0 into NaN.  Each matrix holds other values, so a batch offset that wraps, stops
    early or reads another product's copy of B shows."""
    guard("strided CSR SpMM batch", 64 << 20)
    off, col, _ = a_matrix(0)
    nnz = A_OFF[-1]
    row = torch.searchsorted(off, torch.arange(nnz, device="cuda"), right=True) - 1
    V = batched((nnz,), 9)
    Adense = torch.zeros(BATCH, A_ROWS, A_COLS, dtype=torch.int64, device="cuda")
    Adense[:, row, col] = V
    Bc = batched((A_COLS, N_B), 10)
    Bs = as_dt(Bc.transpose(1, 2).reshape(-1), dt)
    C0 = torch.full((BATCH * A_ROWS * N_B,), float("nan"), dtype=TD[dt], device="cuda")
    arrays = dict(off=off.int(), col=col.int().repeat(BATCH), val=as_dt(V.reshape(-1), dt), nnz=nnz)
    api.set_option("B200SPMV_GENERIC", "all")
    try:
        before = api.stats()
        Cb = cs.spmm(api, A_ROWS, A_COLS, arrays, Bs, C0, LM.ALPHA, 0.0, n=N_B, alg=cs.CUSPARSE_SPMM_CSR_ALG2, batches=BATCH,
                     colval_stride=nnz, compute=cs._VT[TD[dt]], preprocess=False)
        torch.cuda.synchronize()
        after = api.stats()
    finally:
        api.set_option("B200SPMV_GENERIC", "csr")
    assert after["native"] == before["native"] + 1 and after["forwarded"] == before["forwarded"]
    exact(Cb.view(BATCH, N_B, A_ROWS).transpose(1, 2), LM.ALPHA * bmm(Adense, Bc))
    del Cb, C0, Bs, arrays
    release(f"csr spmm batch dt={dt}")
    release(f"strided batches dt={dt}")


# ============================================================================================================ B. 32-bit counts
def spmv_shim(cs, api, op, make_mat, x, y, beta):
    """one cusparseSpMV call sequence (bufferSize, preprocess, SpMV) on caller tensors, the matrix descriptor from make_mat(api);
    returns (stats, last CSR kernel, buffer size) -- the stats and the kernel are the shim's, meaningful for api.impl == "b200"."""
    h = api.cusparseCreate()
    mat = make_mat(api)
    vx, vy = api.cusparseCreateDnVec(x.numel(), x), api.cusparseCreateDnVec(y.numel(), y)
    ct = cs._VT[x.dtype]
    try:
        size = api.cusparseSpMV_bufferSize(h, op, LM.ALPHA, mat, vx, beta, vy, ct)
        buf = torch.empty(max(size, 16), dtype=torch.uint8, device="cuda")
        api.cusparseSpMV_preprocess(h, op, LM.ALPHA, mat, vx, beta, vy, ct, 0, buf)
        api.reset_stats()
        api.cusparseSpMV(h, op, LM.ALPHA, mat, vx, beta, vy, ct, 0, buf)
        torch.cuda.synchronize()
        return api.stats(), api.last_csr_kernel(), size
    finally:
        api.cusparseDestroySpMat(mat)
        api.cusparseDestroyDnVec(vx)
        api.cusparseDestroyDnVec(vy)
        api.cusparseDestroy(h)


def csr(rows, cols, nnz, off, col, val):
    return lambda api: api.cusparseCreateCsr(rows, cols, nnz, off, col, val)


def csr_plan_bytes(N, rows, nnz):
    return LM.round_up_256(N.b200spmv_csr_workspace_bytes(rows, nnz)) + N.b200spmv_csr_flat_workspace_bytes(rows, nnz) + 256


ROWS_BAND = [M - 65, M - 64, M - 2, M - 1]


@pytest.mark.parametrize("rows", ROWS_BAND, ids=["largest_fast", "first_band", "short_refused_before", "flat_refused_before"])
def test_csr_spmv_rows_at_the_int32_limit(N, api, cs, rows):
    """rows near INT32_MAX, 320 entries in the first and the last 10 rows (<= 32 per row: the short kernel's class).  Up to
    INT32_MAX - 65 the specialised kernels serve it (short kernel); above, csr_generic_kernel.  Before the FAST limit matched
    the entry points, INT32_MAX - 2 reached the short kernel, which refused it (INVALID_VALUE, still counted as native).  No call of
    the closed library is made here: its cusparseSpMV (the libcusparse.so.12 that torch ships) made an illegal memory access on this 32-bit CSR at
    rows = INT32_MAX - 65, so it is no reference at these sizes (DESIGN.md 3.11)."""
    nnz, cols = 320, 1024
    kernel = "b200::csr_short_kernel<float>" if rows < M - 64 else "b200::csr_generic_kernel"
    guard(f"spmv rows={rows}", (rows + 1) * 4 + rows * 4 + csr_plan_bytes(N, rows, nnz) + (64 << 20))
    off = torch.empty(rows + 1, dtype=torch.int32, device="cuda")
    off[:11] = torch.arange(0, 176, 16, dtype=torch.int32, device="cuda")
    off[11:rows - 9] = 160
    off[rows - 9:] = torch.arange(176, 336, 16, dtype=torch.int32, device="cuda")
    k = torch.arange(nnz, dtype=torch.int64, device="cuda")
    col, val = LM.col_at(k, cols).int(), LM.val_at(k).float()
    x = LM.fill(torch.empty(cols, dtype=torch.float32, device="cuda"), LM.x_at)
    y = torch.full((rows,), float("nan"), dtype=torch.float32, device="cuda")
    st, kern, _ = spmv_shim(cs, api, 0, csr(rows, cols, nnz, off, col, val), x, y, 0)
    assert (st["native"], st["forwarded"]) == (1, 0), st
    assert kern == kernel, kern
    # the stored rows against the reference of the 20-row matrix; every other row is alpha * 0
    small_off = torch.tensor(LM.offsets("ends", 20, nnz).tolist(), dtype=torch.int64, device="cuda")
    want = LM.reference(small_off, col, val, x, 20)
    exact(y[:10], want[:10])
    exact(y[rows - 10:], want[10:])
    mid = y[10:rows - 10]
    assert not torch.isnan(mid).any() and int(torch.count_nonzero(mid)) == 0
    del off, y, mid
    release(f"spmv rows={rows}")


@pytest.fixture(scope="class")
def big_colval():
    """col (int32, base 0) and val (fp32) of nnz = 2^31 + 2^20 entries, on the device for the cases of TestLargestCounts only: they
    take prefixes of them (INT32_MAX - 65537 and INT32_MAX - 65536 entries, a Sliced-ELL of 2^31 - 65536 slots) or the whole (row
    or slice offsets past 2^31)"""
    guard("col / val of 2^31 + 2^20 entries", BIG * 8 + (8 << 30))
    col = LM.fill(torch.empty(BIG, dtype=torch.int32, device="cuda"), lambda k: LM.col_at(k, COLS_B))
    val = LM.fill(torch.empty(BIG, dtype=torch.float32, device="cuda"), LM.val_at)
    torch.cuda.synchronize()
    yield col, val
    del col, val
    gc.collect()
    torch.cuda.empty_cache()


# profile -> (offsets kind, rows, opA, kernel the call must reach)
PROFILES = {
    "skewed_flat": ("skewed", 1 << 22, 0, "b200::csr_flat_kernel<float>"),
    "uniform_tile": ("uniform", NNZ_FAST // 20, 0, "b200::csr_tile_kernel<float>"),
    "short": ("uniform", -(-NNZ_FAST // 15), 0, "b200::csr_short_kernel<float>"),
    "transpose": ("uniform", NNZ_FAST // 20, 1, "b200::csr_transpose_kernel<float>"),
}
SELL_WIDTH = 16


class TestLargestCounts:
    """The cases that share big_colval's 17 GB; it is freed when the last of them ends."""

    @pytest.mark.parametrize("nnz", [NNZ_FAST, NNZ_FAST + 1], ids=["largest_fast", "first_generic"])
    @pytest.mark.parametrize("profile", list(PROFILES))
    def test_csr_spmv_at_the_nnz_limit(self, N, api, cs, big_colval, profile, nnz):
        kind, rows, op, kernel = PROFILES[profile]
        if nnz > NNZ_FAST:
            kernel = "b200::csr_generic_transpose_kernel" if op else "b200::csr_generic_kernel"
        col, val = big_colval
        n_in, n_out = (rows, COLS_B) if op else (COLS_B, rows)
        plan = csr_plan_bytes(N, rows, nnz)
        guard(f"spmv {profile} nnz={nnz}", (rows + 1) * (4 + 8) + (n_in + 2 * n_out) * 4 + 2 * n_out * 8 + plan + 2 * LM.CHUNK * 8 * 4)
        off64 = LM.offsets(kind, rows, nnz, "cuda")
        assert LM.bound_ok(off64, LM.spread_fan_in(nnz, COLS_B))
        x = LM.fill(torch.empty(n_in, dtype=torch.float32, device="cuda"), LM.x_at)
        off32 = off64.int()
        for beta in (0, LM.BETA):
            y0 = LM.fill(torch.empty(n_out, dtype=torch.int64, device="cuda"), LM.y0_at)
            y = torch.full((n_out,), float("nan"), dtype=torch.float32, device="cuda") if beta == 0 else y0.float()
            st, k, size = spmv_shim(cs, api, op, csr(rows, COLS_B, nnz, off32, col[:nnz], val[:nnz]), x, y, beta)
            assert (st["native"], st["forwarded"]) == (1, 0), st
            assert k == kernel, (k, kernel)
            exact(y, LM.reference(off64, col, val, x, n_out, bool(op), 0, y0 if beta else None))
            del y, y0
        del off64, off32, x
        release(f"spmv {profile} nnz={nnz}")

    @pytest.mark.parametrize("kernel", ["tile", "seg"])
    def test_coo_spmv_at_the_nnz_limit(self, N, api, cs, big_colval, kernel):
        """COO SpMV through the shim at nnz = INT32_MAX - 65537 on coo_tile_kernel and on the segmented kernel
        (B200SPMV_COO_KERNEL), ~20 entries per row, row indices sorted"""
        col, val = big_colval
        nnz, rows = NNZ_FAST, NNZ_FAST // 20
        ws = N.b200spmv_coo_workspace_bytes(rows, nnz)
        guard(f"coo spmv {kernel}", nnz * 4 + (rows + 1) * 8 + rows * (4 + 8) + COLS_B * 4 + ws + 2 * LM.CHUNK * 8 * 4)
        off64 = LM.offsets("uniform", rows, nnz, "cuda")
        row = LM.fill(torch.empty(nnz, dtype=torch.int32, device="cuda"), lambda k: torch.searchsorted(off64, k, right=True) - 1)
        x = LM.fill(torch.empty(COLS_B, dtype=torch.float32, device="cuda"), LM.x_at)
        y = torch.full((rows,), float("nan"), dtype=torch.float32, device="cuda")
        api.set_option("B200SPMV_COO_KERNEL", kernel)
        try:
            st, _, _ = spmv_shim(cs, api, 0, lambda a: a.cusparseCreateCoo(rows, COLS_B, nnz, row, col[:nnz], val[:nnz]), x, y, 0)
        finally:
            api.set_option("B200SPMV_COO_KERNEL", "auto")
        assert (st["native"], st["forwarded"]) == (1, 0), st
        exact(y, LM.reference(off64, col, val, x, rows))
        del row, off64, x, y
        release(f"coo spmv nnz={nnz} {kernel}")

    @pytest.mark.parametrize("slice_size", [32, 7])
    def test_sell_spmv_at_the_nnz_limit(self, N, api, cs, big_colval, slice_size):
        """Sliced-ELL SpMV through the shim with nnz = INT32_MAX - 65537 stored entries: every slice 16 wide, the last row of the
        last slice two short (its two padding slots carry column -1 for the call and get their column back afterwards)"""
        col, val = big_colval
        S, w = slice_size, SELL_WIDTH
        nslices = -(-NNZ_FAST // (S * w))
        vsize, rows = nslices * S * w, nslices * S
        pad = [(nslices - 1) * S * w + j * S + (S - 1) for j in range(w - (vsize - NNZ_FAST), w)]
        assert vsize - NNZ_FAST == len(pad) == 2 and vsize <= BIG
        ws = N.b200spmv_sell_workspace_bytes(rows, vsize, S)
        guard(f"sell spmv S={S}", (nslices + 1) * 4 + rows * (4 + 8) + COLS_B * 4 + ws + 2 * LM.CHUNK * 8 * 4)
        soff = (torch.arange(nslices + 1, dtype=torch.int64, device="cuda") * (S * w)).int()
        x = LM.fill(torch.empty(COLS_B, dtype=torch.float32, device="cuda"), LM.x_at)
        y = torch.full((rows,), float("nan"), dtype=torch.float32, device="cuda")
        col[pad] = -1
        try:
            st, _, _ = spmv_shim(cs, api, 0, lambda a: a.cusparseCreateSlicedEll(rows, COLS_B, NNZ_FAST, vsize, S, soff, col[:vsize],
                                                                                val[:vsize]), x, y, 0)
            assert (st["native"], st["forwarded"]) == (1, 0), st
            exact(y, LM.reference_entries(vsize, LM.sell_row_col(col, S, w), val, x, rows))
        finally:
            col[pad] = LM.col_at(torch.tensor(pad, device="cuda"), COLS_B).int()
        del soff, x, y
        release(f"sell spmv S={S}")

    def test_generic_csr_offsets_past_2_31(self, N, big_colval):
        """CSR 64/32 with nnz = 2^31 + 2^20: int64 row offsets past 2^31 over the skewed profile, fp32 A with fp32 and with fp64
        x / y, beta = 0 into NaN"""
        col, val = big_colval
        rows = 1 << 22
        guard("generic nnz=2^31+2^20", (rows + 1) * 8 + (COLS_B + rows) * 8 + rows * 16 + 2 * LM.CHUNK * 8 * 4)
        off = LM.offsets("skewed", rows, BIG, "cuda")
        assert int(off[-1]) == BIG and LM.bound_ok(off, LM.spread_fan_in(BIG, COLS_B))
        want = LM.reference(off, col, val, LM.fill(torch.empty(COLS_B, dtype=torch.int64, device="cuda"), LM.x_at), rows)
        for xy_dt in (0, 1):
            xt = TD[xy_dt]
            x = LM.fill(torch.empty(COLS_B, dtype=xt, device="cuda"), LM.x_at)
            y = torch.full((rows,), float("nan"), dtype=xt, device="cuda")
            pa, _ka = scal(LM.ALPHA, xy_dt)
            pb, _kb = scal(0, xy_dt)
            rc = N.b200spmv_csr_generic_mv(stream(), 1, 0, 0, xy_dt, 0, rows, COLS_B, BIG, off.data_ptr(), col.data_ptr(),
                                           val.data_ptr(), 0, pa, pb, 0, x.data_ptr(), y.data_ptr())
            torch.cuda.synchronize()
            assert rc == 0, rc
            exact(y, want)
            del x, y
        del off, want
        release("generic nnz=2^31+2^20")

    @pytest.mark.parametrize("op", [0, 1], ids=["N", "T"])
    def test_generic_sell_slice_offsets_past_2_31(self, N, big_colval, op):
        """b200spmv_sell_generic_mv (the route is opt-in: B200SPMV_GENERIC=all) with 2^31 + 2^20 slots: slices of 32 rows x 512,
        int64 slice offsets past 2^31, 32-bit columns; fp32 and fp32-A / fp64-xy, beta = 0 into NaN"""
        col, val = big_colval
        S, w = 32, 512
        nslices = BIG // (S * w)
        rows = nslices * S
        assert nslices * S * w == BIG
        n_in, n_out = (rows, COLS_B) if op else (COLS_B, rows)
        guard(f"generic sell op={op}", (nslices + 1) * 8 + (n_in + n_out) * 8 + n_out * 8 + 2 * LM.CHUNK * 8 * 4)
        soff = torch.arange(nslices + 1, dtype=torch.int64, device="cuda") * (S * w)
        want = LM.reference_entries(BIG, LM.sell_row_col(col, S, w), val,
                                    LM.fill(torch.empty(n_in, dtype=torch.int64, device="cuda"), LM.x_at), n_out, bool(op))
        for xy_dt in (0, 1):
            xt = TD[xy_dt]
            x = LM.fill(torch.empty(n_in, dtype=xt, device="cuda"), LM.x_at)
            y = torch.full((n_out,), float("nan"), dtype=xt, device="cuda")
            pa, _ka = scal(LM.ALPHA, xy_dt)
            pb, _kb = scal(0, xy_dt)
            rc = N.b200spmv_sell_generic_mv(stream(), 1, 0, 0, xy_dt, op, rows, COLS_B, S, soff.data_ptr(), col.data_ptr(),
                                            val.data_ptr(), 0, pa, pb, 0, x.data_ptr(), y.data_ptr())
            torch.cuda.synchronize()
            assert rc == 0, rc
            exact(y, want)
            del x, y
        del soff, want
        release(f"generic sell op={op}")


# ============================================================================================================ C. 64-bit values
@pytest.mark.parametrize("base", [0, 1])
@pytest.mark.parametrize("op", [0, 1], ids=["N", "T"])
@pytest.mark.parametrize("types", [(0, 0), (0, 1)], ids=["f32", "f32_f64xy"])
@pytest.mark.parametrize("idx", [(1, 1), (1, 0)], ids=["64_64", "64_32"])
def test_generic_csr_columns_past_2_31(N, idx, types, op, base):
    """b200spmv_csr_generic_mv with cols = 2^31 + 2^20 (64-bit columns) or INT32_MAX (32-bit columns: with base 1 the largest
    stored index is still INT32_MAX): entries on column 0, 2^31 - 1 and 2^31 (where they exist) and cols - 1; 4096 rows of ~64"""
    off64_, col64_ = idx
    a_dt, xy_dt = types
    cols = BIG if col64_ else M
    rows, nnz = 4096, 4096 * 64 + 5
    xt, xsz = TD[xy_dt], (8 if xy_dt else 4)
    n_in, n_out = (rows, cols) if op else (cols, rows)
    guard(f"generic cols={cols}", (n_in + n_out) * xsz + nnz * 64 + 2 * LM.CHUNK * 8 * 2)
    off = LM.offsets("uniform", rows, nnz, "cuda")
    k = torch.arange(nnz, dtype=torch.int64, device="cuda")
    col, val = LM.col_at(k, cols), LM.val_at(k)
    offd = (off + base) if off64_ else (off + base).int()
    cold = (col + base) if col64_ else (col + base).int()
    vald = val.to(TD[a_dt])
    x = LM.fill(torch.empty(n_in, dtype=xt, device="cuda"), LM.x_at)
    pa, _ka = scal(LM.ALPHA, xy_dt)
    for beta in (0, LM.BETA):
        pb, _kb = scal(beta, xy_dt)
        y = LM.fill(torch.empty(n_out, dtype=xt, device="cuda"), LM.y0_at) if beta else \
            torch.full((n_out,), float("nan"), dtype=xt, device="cuda")
        rc = N.b200spmv_csr_generic_mv(stream(), off64_, col64_, a_dt, xy_dt, op, rows, cols, nnz, offd.data_ptr(), cold.data_ptr(),
                                       vald.data_ptr(), base, pa, pb, 0, x.data_ptr(), y.data_ptr())
        torch.cuda.synchronize()
        assert rc == 0, rc
        if op == 0:
            y0 = LM.y0_at(torch.arange(rows, device="cuda")) if beta else None
            exact(y, LM.reference(off, col, val, x, rows, False, 0, y0))
        else:
            # A^T x is non-zero on the stored columns only: those against the int64 sums, every other element against beta * y0
            r = torch.searchsorted(off, k, right=True) - 1
            ucol, inv = torch.unique(col, return_inverse=True)
            acc = torch.zeros(ucol.numel(), dtype=torch.int64, device="cuda").index_add_(0, inv, val * x[r].long())
            exact(y[ucol], LM.ALPHA * acc + (LM.BETA * LM.y0_at(ucol) if beta else 0))
            y[ucol] = (LM.BETA * LM.y0_at(ucol)).to(xt) if beta else 0
            for s in range(0, n_out, LM.CHUNK):
                e = min(n_out, s + LM.CHUNK)
                want = LM.BETA * LM.y0_at(torch.arange(s, e, device="cuda")) if beta else torch.zeros(e - s, dtype=torch.int64, device="cuda")
                exact(y[s:e], want)
        del y
    del x, off, col, val, offd, cold, vald
    release(f"generic cols={cols} op={op}")


@pytest.mark.parametrize("xy_dt", [0, 1], ids=["f32", "f32_f64xy"])
def test_generic_coo_rows_past_2_31(N, xy_dt):
    """b200spmv_coo_generic_mv (the route is opt-in: B200SPMV_GENERIC=all) with rows = 2^31 + 2^20 and 64-bit indices: 16 entries on
    each of rows 0-4, 2^31 - 3 ... 2^31 + 2 and the last 9 rows, every other row empty; beta = 0 into NaN"""
    rows, cols, nnz = BIG, 1024, 320
    xt, xsz = TD[xy_dt], (8 if xy_dt else 4)
    guard("generic coo rows=2^31+2^20", rows * xsz + (1 << 30))
    table = torch.tensor(list(range(5)) + list(range(2**31 - 3, 2**31 + 3)) + list(range(BIG - 9, BIG)), dtype=torch.int64,
                         device="cuda")
    k = torch.arange(nnz, dtype=torch.int64, device="cuda")
    row, col, val = table[k // 16], LM.col_at(k, cols), LM.val_at(k).float()
    x = LM.fill(torch.empty(cols, dtype=xt, device="cuda"), LM.x_at)
    y = torch.full((rows,), float("nan"), dtype=xt, device="cuda")
    pa, _ka = scal(LM.ALPHA, xy_dt)
    pb, _kb = scal(0, xy_dt)
    rc = N.b200spmv_coo_generic_mv(stream(), 1, 0, xy_dt, rows, cols, nnz, row.data_ptr(), col.data_ptr(), val.data_ptr(), 0, pa, pb, 0,
                                   x.data_ptr(), y.data_ptr())
    torch.cuda.synchronize()
    assert rc == 0, rc
    want = torch.zeros(table.numel(), dtype=torch.int64, device="cuda").index_add_(0, k // 16, val.long() * x[col].long())
    exact(y[table], LM.ALPHA * want)
    y[table] = 0
    assert not torch.isnan(y).any() and int(torch.count_nonzero(y)) == 0
    del y, x
    release(f"generic coo xy_dt={xy_dt}")
