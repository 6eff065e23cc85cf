"""CPU: what tests/test_limits_gpu.py relies on.  The closed-form generators and the chunked int64 reference of oracle/limits.py
against scipy at small sizes (and the exactness bound: no partial sum at or above 2^24), the boundary values of the SpMV route
through the exported b200spmv_route predicate, and the host-side workspace sizes the GPU file's memory guard adds up."""
import ctypes as C

import numpy as np
import pytest
import scipy.sparse as sp
import torch

from cudalibrarysamples_b200.lib import load
from oracle import limits as LM

CSR, COO, SELL = 1, 3, 7
N, T = 0, 1
I32, I64 = 2, 3
F32, F64 = 0, 1
FORWARD, FAST, GENERIC = 0, 1, 2
M = LM.INT32_MAX
NNZ_FAST = M - 65537                  # the largest nnz the specialised SpMV kernels take


@pytest.fixture()
def lib(built_lib):
    L = load(built_lib)
    yield L
    assert L.b200spmv_set_option(b"B200SPMV_GENERIC", b"csr") == 0      # back to the default


def route(L, fmt=CSR, op=N, rows=1000, cols=1000, nnz=16000, vt=F32):
    return L.b200spmv_route(fmt, op, 0, I32, I32, vt, vt, vt, vt, C.c_int64(rows), C.c_int64(cols), C.c_int64(nnz))


# ---- generators and reference ---------------------------------------------------------------------------------------------------
def scipy_ref(off, col, val, x, rows, cols, transpose, y0):
    A = sp.csr_matrix((val.numpy().astype(np.float64), col.numpy(), off.numpy()), shape=(rows, cols))
    y = (A.T if transpose else A) @ x.numpy().astype(np.float64)
    return LM.ALPHA * y + (0 if y0 is None else LM.BETA * y0.numpy())


@pytest.mark.parametrize("kind,rows,nnz", [("uniform", 997, 20 * 997 + 13), ("skewed", 1 << 12, 512 << 12), ("ends", 300, 320)])
@pytest.mark.parametrize("transpose", [False, True])
@pytest.mark.parametrize("base", [0, 1])
def test_reference_matches_scipy(kind, rows, nnz, transpose, base, monkeypatch):
    monkeypatch.setattr(LM, "CHUNK", 1000)                  # several chunks, one ragged
    cols = 3001
    off = LM.offsets(kind, rows, nnz)
    assert off.shape == (rows + 1,) and int(off[0]) == 0 and int(off[-1]) == nnz and bool((off[1:] >= off[:-1]).all())
    lens = off[1:] - off[:-1]
    assert int(lens[0]) > 0 and int(lens[-1]) > 0 and int((lens == 0).sum()) >= 1      # first and last row stored, an empty row
    col = LM.fill(torch.empty(nnz, dtype=torch.int64), lambda k: LM.col_at(k, cols) + base)
    val = LM.fill(torch.empty(nnz, dtype=torch.float32), LM.val_at)
    assert int(col.min()) == base and int(col.max()) == cols - 1 + base and bool((val != 0).all())
    assert set(val.unique().tolist()) <= {-3.0, -2.0, -1.0, 1.0, 2.0, 3.0}
    n_in, n_out = (rows, cols) if transpose else (cols, rows)
    x = LM.fill(torch.empty(n_in, dtype=torch.float64), LM.x_at)
    y0 = LM.fill(torch.empty(n_out, dtype=torch.int64), LM.y0_at)
    fan = int(torch.bincount(col - base).max())
    assert fan <= LM.spread_fan_in(nnz, cols) and LM.bound_ok(off, fan)
    for y0_ in (None, y0):
        got = LM.reference(off, col, val, x, n_out, transpose, base, y0_)
        want = scipy_ref(off, col - base, val, x, rows, cols, transpose, y0_)
        np.testing.assert_array_equal(got.numpy(), want)
        # every partial sum of any order is below 2^24: the sum of |products| and |alpha * that| + |beta * y0| are
        A = sp.csr_matrix((np.abs(val.numpy()).astype(np.float64), (col - base).numpy(), off.numpy()), shape=(rows, cols))
        absum = (A.T if transpose else A) @ np.abs(x.numpy())
        assert (abs(LM.ALPHA) * absum + abs(LM.BETA) * 3).max() < 2**24


def test_col_at_reaches_the_index_extremes():
    k = torch.arange(8, dtype=torch.int64)
    big = 2**31 + 2**20
    c = LM.col_at(k, big)
    assert c[0] == 0 and c[1] == big - 1 and c[2] == 2**31 - 1 and c[3] == 2**31
    c = LM.col_at(k, M)                                     # int32 columns with base 1 still fit: the largest is M - 1
    assert c[1] == M - 1 and int(c.max()) <= M - 1


def test_group_b_profiles_keep_the_bounds():
    """the row lengths the GPU file builds at the largest FAST nnz: short rows <= 32 with one row > 32 nowhere, uniform rows with
    one row past 32 (tile kernels, not the short one), skewed rows <= 2048; column fan-in within the A^T bound"""
    for kind, rows, lo, hi in (("uniform", -(-NNZ_FAST // 15), 15, 32), ("uniform", NNZ_FAST // 20, 33, 64), ("skewed", 1 << 22, 900, 2048)):
        off = LM.offsets(kind, rows, NNZ_FAST)
        assert int(off[-1]) == NNZ_FAST and lo <= LM.max_row(off) <= hi, (kind, rows, LM.max_row(off))
        assert LM.bound_ok(off, LM.spread_fan_in(NNZ_FAST + 1, 1 << 21))


# ---- routing at the 32-bit edges --------------------------------------------------------------------------------------------
def test_fast_row_limit(lib):
    """the specialised kernels take rows, cols <= INT32_MAX - 64; the band above runs on csr_generic_kernel (64-bit arithmetic)"""
    assert route(lib, rows=M - 65, nnz=320) == FAST
    assert route(lib, cols=M - 65) == FAST
    for rows in (M - 64, M - 2, M - 1):
        assert route(lib, rows=rows, nnz=320) == GENERIC, rows
        assert route(lib, op=T, rows=rows, nnz=320) == GENERIC, rows
    assert route(lib, cols=M - 64) == GENERIC
    assert route(lib, op=T, cols=M - 64) == GENERIC
    # COO / Sliced-ELL in the band: the generic kernels serve them only under B200SPMV_GENERIC=all
    assert route(lib, COO, rows=M - 65, nnz=320) == FAST and route(lib, COO, rows=M - 64, nnz=320) == FORWARD
    assert lib.b200spmv_set_option(b"B200SPMV_GENERIC", b"all") == 0
    assert route(lib, COO, rows=M - 64, nnz=320) == GENERIC and route(lib, SELL, rows=M - 1, nnz=320) == GENERIC
    assert lib.b200spmv_set_option(b"B200SPMV_GENERIC", b"off") == 0
    assert route(lib, rows=M - 64, nnz=320) == FORWARD


def test_fast_nnz_limit(lib):
    for vt in (F32, F64):
        for fmt in (CSR, COO, SELL):
            assert route(lib, fmt, rows=1 << 22, nnz=NNZ_FAST, vt=vt) == FAST
        assert route(lib, rows=1 << 22, nnz=NNZ_FAST + 1, vt=vt) == GENERIC
        assert route(lib, op=T, rows=1 << 22, nnz=NNZ_FAST, vt=vt) == FAST


# ---- workspace sizes of the memory guard ------------------------------------------------------------------------------------
def test_spmm_csr_workspace_is_the_row_major_copy_of_b(lib):
    for dt, vsz in ((F32, 4), (F64, 8)):
        for n in (32 * 65535, 32 * 65535 + 1, 64 * 65535 - 1):
            assert lib.b200spmm_csr_workspace_bytes(dt, 3, n, 0) == LM.round_up_256(3 * n * vsz)
            assert lib.b200spmm_csr_workspace_bytes(dt, 3, n, 1) == 0       # row-major B is read in place


def test_spmv_plan_sizes_at_the_largest_fast_nnz(lib):
    """tile plan + flat plan of the largest profiles: positive, growing with nnz, and bounded -- the flat plan holds a 32-bit copy
    of col_ind (hot-column slots), so about nnz * 4 bytes plus its bit masks; with the 17 GB of col / val a case stays near 30 GB"""
    for rows in (-(-NNZ_FAST // 15), NNZ_FAST // 20, 1 << 22):
        tile = lib.b200spmv_csr_workspace_bytes(rows, NNZ_FAST)
        flat = lib.b200spmv_csr_flat_workspace_bytes(rows, NNZ_FAST)
        assert 0 < tile < 4e9 and NNZ_FAST * 4 <= flat < NNZ_FAST * 5, (rows, tile, flat)
        assert lib.b200spmv_csr_flat_workspace_bytes(rows, NNZ_FAST // 2) < flat
    tile = lib.b200spmv_csr_workspace_bytes(M - 65, 320)
    assert 0 < tile < 4e9


@pytest.mark.parametrize("slice_size,transpose", [(32, False), (7, False), (7, True)])
def test_sell_entry_reference_matches_scipy(slice_size, transpose, monkeypatch):
    """reference_entries over a Sliced-ELL layout (sell_row_col), padding slots (column -1) skipped, against scipy"""
    monkeypatch.setattr(LM, "CHUNK", 1000)
    S, w, nslices, cols = slice_size, 16, 37, 501
    vsize, rows = nslices * S * w, nslices * S
    col = LM.fill(torch.empty(vsize, dtype=torch.int32), lambda k: LM.col_at(k, cols))
    val = LM.fill(torch.empty(vsize, dtype=torch.float32), LM.val_at)
    pad = [(nslices - 1) * S * w + j * S + (S - 1) for j in (w - 2, w - 1)]
    col[pad] = -1
    i = np.arange(vsize)
    r = (i // (S * w)) * S + (i % (S * w)) % S
    live = col.numpy() >= 0
    A = sp.csr_matrix((val.numpy()[live].astype(np.float64), (r[live], col.numpy()[live])), shape=(rows, cols))
    n_in, n_out = (rows, cols) if transpose else (cols, rows)
    x = LM.fill(torch.empty(n_in, dtype=torch.int64), LM.x_at)
    want = LM.ALPHA * ((A.T if transpose else A) @ x.numpy().astype(np.float64))
    got = LM.reference_entries(vsize, LM.sell_row_col(col, S, w), val, x, n_out, transpose, device="cpu")
    np.testing.assert_array_equal(got.numpy(), want)
    assert int(np.bincount(r[live]).max()) == w and int(np.bincount(r[live], minlength=rows)[-1]) == w - 2
