"""CPU: B200SPMV_ZCSR -- `on` sends every call of b200spmv_csr_z's class to it and nothing outside the class, `auto` restores the
measured route, an unknown value is refused; and the complex kernel's split walk keeps the write-once structure of the walk model at
its own chunk size."""
import ctypes as C

import numpy as np
import pytest

from cudalibrarysamples_b200.lib import load
from oracle import spmv_csr_z_ref as R

F32, F64, F16, C32, C64 = 0, 1, 2, 4, 5
CSR, COO, SELL, CSC = 1, 2, 9, 3
I32, I64 = 2, 3
FORWARD, FAST, ZCSR = 0, 1, 4


def route(L, fmt=CSR, op=0, alg=0, off=I32, col=I32, a=C64, x=None, y=None, compute=None, rows=1 << 20, cols=1 << 20, nnz=16 << 20):
    x = a if x is None else x
    y = a if y is None else y
    compute = a if compute is None else compute
    return L.b200spmv_route(fmt, op, alg, off, col, a, x, y, compute, C.c_int64(rows), C.c_int64(cols), C.c_int64(nnz))


def test_zcsr_option_switches_the_class_and_only_the_class(built_lib):
    from scripts.spmv_csr_z_bench import NATIVE
    nat = eval(NATIVE)
    L = load(built_lib)
    assert L.b200spmv_set_option(b"B200SPMV_ZCSR", b"sometimes") == -1
    assert L.b200spmv_set_option(b"B200SPMV_ZCSR", b"on") == 0
    try:
        for op in (0, 1, 2):
            for rows, nnz in ((1000, 16000), (1 << 20, 16 << 20), (0, 0), (5, 25)):
                ok = dict(op=op, rows=rows, cols=rows, nnz=nnz)
                for alg in (0, 2, 3):
                    assert route(L, alg=alg, **ok) == ZCSR, (op, rows, alg)
                assert route(L, a=C32, **ok) == FORWARD and route(L, a=C32, x=C64, y=C64, compute=C64, **ok) == FORWARD
                assert route(L, compute=C32, **ok) == FORWARD and route(L, y=C32, **ok) == FORWARD
                assert route(L, off=I64, col=I64, **ok) == FORWARD and route(L, col=I64, **ok) == FORWARD
                for fmt in (COO, SELL, CSC):
                    assert route(L, fmt=fmt, **ok) == FORWARD
                for alg in (1, 4, 5):
                    assert route(L, alg=alg, **ok) == FORWARD
            assert route(L, op=op, rows=1 << 31, cols=1 << 20, nnz=16 << 31) == FORWARD
        assert route(L, a=F32) == FAST and route(L, a=F64) == FAST
    finally:
        assert L.b200spmv_set_option(b"B200SPMV_ZCSR", b"auto") == 0
    for op in (0, 1, 2):
        want = ZCSR if nat(op, 1 << 20, 1 << 20, 16 << 20) else FORWARD
        assert route(L, op=op) == want


@pytest.mark.parametrize("lengths", [[0, 1, 255, 256, 257, 0, 511, 513, 3, 10257, 0], [1, 2, 3, 0, 30, 31, 32, 33] * 40, [1000]])
def test_split_walk_model_at_the_complex_chunk_size(built_lib, lengths):
    """at b200spmv_csr_z's E: every row written once, every carry slot written once and read once by one fix-up at the row's first
    chunk, and both walks add the same pieces"""
    E = R.params(load(built_lib))["chunk"]
    off = np.concatenate([[0], np.cumsum(lengths)]).astype(np.int64)
    nch = max(1, -(-int(off[-1]) // E))
    sw, sr, sp = R.walk(off, E, split=True)
    uw, _, up = R.walk(off, E, split=False)
    for writes in (sw, uw):
        assert sorted(w[1] for w in writes if w[0] == "y") == list(range(len(lengths)))
    slots = [w[1] for w in sw if w[0] == "carry"]
    assert len(slots) == len(set(slots)) and all(s < 2 * nch for s in slots)
    assert sorted(r[1] for r in sr) == sorted(slots)
    for _, s, r, c in sr:
        assert int(off[r]) // E == c and s in (R.slot("out", c),) + tuple(R.slot("in", c2) for c2 in range(c + 1, nch))
    assert sorted((p[0], p[1], p[2]) for p in sp) == sorted((p[0], p[1], p[2]) for p in up)
