"""CPU: the sparse <-> dense restatement (oracle/dense_ref.py) against scipy and the three reference samples' own arrays, its
window / ld / base edges and the pinned zero predicate, and b200dense_route's table: one case per forwarding reason."""
import numpy as np
import pytest
import scipy.sparse as sp

from oracle import dense_ref as R

ROW, COL = R.ORDER_ROW, R.ORDER_COL


def f32(a):
    return np.asarray(a, np.float32).view(np.uint8).reshape(-1, 4)


def test_samples_round_trip_against_their_goldens():
    S = R.samples()
    s = S["sparse2dense_csr"]
    out = R.csr_to_dense(np.zeros((20, 4), np.uint8), 5, 4, 4, ROW, s["csr_offsets"], s["csr_columns"], f32(s["csr_values"]))
    assert out.view(np.float32).ravel().tolist() == s["dense_result"]
    s = S["dense2sparse_csr"]
    off, ind, val = R.dense_to_csr(f32(s["dense"]), 5, 4, 4, ROW, 4)
    assert off.tolist() == s["csr_offsets_result"] and ind.tolist() == s["csr_columns_result"]
    assert val.view(np.float32).ravel().tolist() == s["csr_values_result"]
    s = S["dense2sparse_blockedell"]
    ev = R.dense_to_bell(f32(s["dense"]), 4, 6, 6, ROW, 2, s["ell_columns"], np.full((16, 4), 0xFF, np.uint8))
    assert ev.view(np.float32).ravel().tolist() == s["ell_values_result"]        # the -1 slot holds zeros


@pytest.mark.parametrize("order", [ROW, COL])
@pytest.mark.parametrize("base", [0, 1])
@pytest.mark.parametrize("csc", [False, True])
def test_against_scipy_with_ld_padding(order, base, csc):
    rng = np.random.default_rng(order * 4 + base * 2 + csc)
    m, n = 23, 17
    A = sp.random(m, n, density=0.3, format="csr", random_state=rng, dtype=np.float64)
    A.data[::5] = 0.0                                      # explicit zeros vanish on the way back
    ld = (n if order == ROW else m) + 3
    size = ld * (m if order == ROW else n)
    init = rng.integers(0, 256, (size, 8), dtype=np.uint8)
    S = A.tocsc() if csc else A
    dense = R.csr_to_dense(init, m, n, ld, order, S.indptr + base, S.indices + base, S.data.view(np.uint8).reshape(-1, 8), base, csc)
    D = dense.reshape(-1).view(np.float64)
    win = R.window(m, n, ld, order)
    assert np.array_equal(D[win], A.toarray())
    outside = np.ones(size, bool)
    outside[win.ravel()] = False
    assert np.array_equal(dense[outside], init[outside])  # the ld padding untouched
    off, ind, val = R.dense_to_csr(dense, m, n, ld, order, 8, base, csc)
    B = A.copy()
    B.eliminate_zeros()
    B = B.tocsc() if csc else B
    B.sort_indices()
    assert np.array_equal(off - base, B.indptr) and np.array_equal(ind - base, B.indices)
    assert np.array_equal(val.view(np.float64).ravel(), B.data)


def test_zero_predicate():
    f32v = np.array([0.0, -0.0, 1e-45, np.nan, np.inf, -1.0], np.float32)
    assert R.nonzero(f32v.view(np.uint8).reshape(-1, 4), 4).tolist() == [False, False, True, True, True, True]
    f16 = np.array([0.0, -0.0, 6e-8, np.nan, np.inf, 1.0], np.float16)
    assert R.nonzero(f16.view(np.uint8).reshape(-1, 2), 2).tolist() == [False, False, True, False, True, True]
    # bf16 bits read as fp16: 0x7C00 (about 2.6e36) kept, anything larger (0x7C01, Inf 0x7F80, NaN 0x7FC1) zero
    bf16 = np.array([0x0000, 0x8000, 0x0001, 0x7C00, 0xFC01, 0x7F80, 0x7FC1, 0x3F80], np.uint16)
    assert R.nonzero(bf16.view(np.uint8).reshape(-1, 2), 2).tolist() == [False, False, True, True, False, False, False, True]
    z = np.array([0, complex(-0.0, 0.0), complex(0, 1e-320), complex(np.nan, 0)], np.complex128)
    assert R.nonzero(z.view(np.uint8).reshape(-1, 16), 8).tolist() == [False, False, True, True]


def test_duplicates_last_wins_and_out_of_range_skipped():
    dense = np.zeros((6, 4), np.uint8)
    vals = f32([1, 2, 3, 4])
    out = R.csr_to_dense(dense, 2, 3, 3, ROW, [0, 3, 4], [1, 1, 5, -1], vals)
    assert out.view(np.float32).ravel().tolist() == [0, 2, 0, 0, 0, 0]


# b200dense_route(direction, format, order, vtype, off_type, col_type, base, rows, cols, nnz, batch, alg, bs)
S2D, D2S, CSR, CSC, COO, BELL, BSR = 0, 1, 1, 2, 3, 5, 6
I32, I64 = 2, 3
ROUTED = (D2S, BELL, ROW, 2, I32, I32, 0, 8192, 8192, 1 << 25, 1, 0, 16)      # dense -> Blocked-ELL, row-major, bs 16, fp16


@pytest.fixture(scope="module")
def L():
    from cudalibrarysamples_b200 import lib
    return lib.shim()


@pytest.mark.parametrize("args", [
    (S2D, CSR, ROW, 0, I64, I64, 0, 100, 100, 10, 1, 0, 0),       # 64-bit indices
    (S2D, CSR, ROW, 0, I32, I32, 2, 100, 100, 10, 1, 0, 0),       # base
    (D2S, CSR, ROW, 10, I32, I32, 0, 100, 100, 10, 1, 0, 0),      # integer values for dense -> sparse
    (D2S, CSR, ROW, 6, I32, I32, 0, 100, 100, 10, 1, 0, 0),       # complex fp16: predicate not pinned
    (D2S, COO, ROW, 0, I32, I32, 0, 100, 100, 10, 1, 0, 0),       # dense -> COO
    (S2D, CSR, COL, 0, I32, I32, 0, 100, 100, 10, 4, 0, 0),       # strided batch
    (S2D, CSR, ROW, 0, I32, I32, 0, 100, 100, 10, 1, 1, 0),       # alg
    (S2D, BSR, ROW, 0, I32, I32, 0, 100, 100, 10, 1, 0, 0),       # format
    (S2D, CSR, 3, 0, I32, I32, 0, 100, 100, 10, 1, 0, 0),         # order
    (S2D, BELL, ROW, 2, I32, I32, 0, 8192, 8192, 1 << 25, 1, 0, 16),   # refused by the closed library
    (S2D, CSR, ROW, 2, I32, I32, 0, 8192, 8192, 1 << 20, 1, 0, 0),     # not measured at parity
    (D2S, CSR, COL, 0, I32, I32, 0, 8192, 8192, 1 << 24, 1, 0, 0),     # not the closed library's index order
    (D2S, BELL, ROW, 2, I32, I32, 0, 8192, 8192, 1 << 25, 1, 0, 32),   # bs 32: slower at 8192^2
    (D2S, BELL, COL, 2, I32, I32, 0, 8192, 8192, 1 << 25, 1, 0, 16),   # column-major: slower
    (D2S, BELL, ROW, 1, I32, I32, 0, 8192, 8192, 1 << 25, 1, 0, 16),   # fp64: not measured
    (D2S, BELL, ROW, 2, I32, I32, 0, 4096, 4096, 1 << 23, 1, 0, 16),   # below the measured sizes
    (D2S, BELL, ROW, 2, I32, I32, 0, 32768, 32768, 1 << 27, 1, 0, 16), # above them
])
def test_route_forwards(L, args):
    assert L.b200dense_route(*args) == 0


def test_route_serves_the_measured_blocked_ell_class(L):
    assert L.b200dense_route(*ROUTED) == 1
    for vt, n in ((0, 16384), (2, 16384)):          # fp32, and the largest measured size
        assert L.b200dense_route(D2S, BELL, ROW, vt, I32, I32, 1, n, n, n * n // 2, 1, 0, 16) == 1


def test_dense_option_switches_every_admitted_call_and_only_those(L):
    try:
        assert L.b200spmv_set_option(b"B200SPMV_DENSE", b"sometimes") == -1
        assert L.b200spmv_set_option(b"B200SPMV_DENSE", b"on") == 0
        for args in ((S2D, CSR, ROW, 2, I32, I32, 0, 8192, 8192, 1 << 20, 1, 0, 0), (S2D, BELL, COL, 0, I32, I32, 1, 64, 64, 2048, 1, 0, 16),
                     (D2S, CSC, ROW, 5, I32, I32, 0, 5, 4, 3, 1, 0, 0), (S2D, COO, ROW, 1, I32, I32, 0, 5, 4, 3, 1, 0, 0)):
            assert L.b200dense_route(*args) == 1, args
        for args in ((S2D, CSR, ROW, 0, I64, I64, 0, 100, 100, 10, 1, 0, 0), (D2S, COO, ROW, 0, I32, I32, 0, 100, 100, 10, 1, 0, 0),
                     (D2S, CSR, ROW, 15, I32, I32, 0, 100, 100, 10, 1, 0, 0), (S2D, CSR, COL, 0, I32, I32, 0, 100, 100, 10, 4, 0, 0)):
            assert L.b200dense_route(*args) == 0, args
    finally:
        assert L.b200spmv_set_option(b"B200SPMV_DENSE", b"auto") == 0
    assert L.b200dense_route(S2D, CSR, ROW, 2, I32, I32, 0, 8192, 8192, 1 << 20, 1, 0, 0) == 0


def test_route_forward_env():
    import os
    import subprocess
    import sys
    code = ("from cudalibrarysamples_b200 import lib; L = lib.shim(); "
            f"print(L.b200dense_route{ROUTED})")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    p = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, cwd=root, env=dict(os.environ, B200SPMV_FORWARD="1"))
    assert p.returncode == 0 and p.stdout.strip() == "0", p.stdout + p.stderr


def test_entry_points_are_exported(L):
    for name in ("b200csr2dense", "b200coo2dense", "b200bell2dense", "b200dense2csr", "b200dense2bell", "b200dense_route",
                 "cusparseSparseToDense", "cusparseDenseToSparse_convert"):
        assert hasattr(L, name), name
