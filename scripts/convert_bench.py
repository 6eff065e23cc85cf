#!/usr/bin/env python
"""Format conversions, ours (convert.cu) against the closed library on the same buffers, in one process (DESIGN.md 3.23).

Matrices: R-MAT 1M and 10M with 16 per row, uniform 2M with 16 per row, the 5-point 8192^2 stencil.  Per matrix:
* csr2csc: SYMBOLIC, then NUMERIC with fp16, fp32, fp64 and complex128 values (b200csr2csc vs cusparseCsr2cscEx2);
* coosort ByRow / ByColumn on the matrix as COO in three input orders: row order, column order and a seeded shuffle (b200coosort vs
  cusparseXcoosortByRow / ByColumn).  The sort is in place, so every timed call first restores the input; that copy is timed on its
  own and taken off both sides;
* coo2csr and csr2coo (b200coo2csr / b200csr2coo vs cusparseXcoo2csr / Xcsr2coo).

Each call is timed with CUDA events after a warm-up, median of three windows.  Reported per row: our time and the closed library's,
the speed-up, the compulsory bytes (inputs read once, outputs written once) over each time, whether the outputs are equal (bit for
bit; coosort's P too), and the verdict of b200conv_route for that call.  The card's name and power limit are read in the same run.
usage: python scripts/convert_bench.py [--quick] [--json out.json]"""
import argparse
import ctypes as C
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from cudalibrarysamples_b200 import cusparse_api as cs  # noqa: E402
from cudalibrarysamples_b200 import lib as _lib  # noqa: E402
from cudalibrarysamples_b200 import workloads as W  # noqa: E402
from scripts.sddmm_bsr_bench import card, timeit  # noqa: E402
from scripts.spmm_csr_t_bench import matrix as csrt_matrix  # noqa: E402

DEV = torch.device("cuda:0")
MATRICES = ("rmat1m", "rmat10m", "uniform2m", "stencil8192")
VALUE_TYPES = (None, torch.float16, torch.float32, torch.float64, torch.complex128)       # None: SYMBOLIC
CSR2CSC, COOSORT_ROW, COOSORT_COL, COO2CSR, CSR2COO = 0, 1, 2, 3, 4

# The classes b200conv_route runs natively (DESIGN.md 3.23), as the predicate the CPU route test evaluates over (op, m, n, nnz, arg:
# csr2csc's value bytes, 0 for SYMBOLIC): coosort ByRow / ByColumn (1 / 2) on the measured sizes, 1M to 8192^2 rows and columns with 4
# to 16 entries per row, where every case ran 1.8x - 5.0x faster.  csr2csc, coo2csr and csr2coo measured below parity (a 1.20x csr2coo
# on the stencil alone does not make a class); the identity permutation was not measured.
NATIVE = "lambda op, m, n, nnz, arg: op in (1, 2) and 1 << 20 <= m <= 8192 ** 2 and 1 << 20 <= n <= 8192 ** 2 and 4 * m <= nnz <= 16 * m"


def matrix(name):
    """(rows, cols, off, col) on the device, int32, base 0, sorted columns"""
    if name == "rmat10m":
        rows = 10 << 20
        off, col, _ = W.rmat_csr(rows, avg_nnz=16, seed=42, val_seed=43, dtype=torch.float32)
        return rows, rows, off.int().contiguous(), col.int().contiguous()
    rows, cols, off, col, _ = csrt_matrix(name)
    return rows, cols, off, col


def ptr(t):
    return C.c_void_p(t.data_ptr()) if t is not None else C.c_void_p(0)


def values(nnz, dt, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    v = torch.randint(-(1 << 15), 1 << 15, (nnz * (2 if dt.is_complex else 1),), device=DEV, generator=g, dtype=torch.int32)
    return (v.double().view(torch.complex128) if dt.is_complex else v.to(dt)).contiguous()


def same(a, b):
    if a is None:
        return b is None
    return bool(torch.equal(a.reshape(-1).view(torch.uint8), b.reshape(-1).view(torch.uint8)))


def csr2csc_case(L, R, h, name, m, n, off, col, dt):
    nnz = col.numel()
    val = None if dt is None else values(nnz, dt, 7)
    width = 0 if dt is None else val.element_size()
    vt = cs.CUDA_R_32F if dt is None else cs._CONV_VT[dt]
    action = cs.CUSPARSE_ACTION_SYMBOLIC if dt is None else cs.CUSPARSE_ACTION_NUMERIC
    outs = [(torch.empty(n + 1, dtype=torch.int32, device=DEV), torch.empty(nnz, dtype=torch.int32, device=DEV),
             None if val is None else torch.empty_like(val)) for _ in range(2)]
    wsb = L.b200csr2csc_workspace_bytes(m, n, nnz)
    ws = torch.empty(wsb, dtype=torch.uint8, device=DEV)
    st = torch.cuda.current_stream().cuda_stream
    o = outs[0]
    ours = lambda: L.b200csr2csc(st, m, n, nnz, ptr(val), ptr(off), ptr(col), ptr(o[2]), ptr(o[0]), ptr(o[1]), width, int(dt is not None), 0,  # noqa: E731
                                 ptr(ws), wsb)
    c = outs[1]
    args = (C.c_int(m), C.c_int(n), C.c_int(nnz), ptr(val), ptr(off), ptr(col), ptr(c[2]), ptr(c[0]), ptr(c[1]), C.c_int(vt),
            C.c_int(action), C.c_int(0), C.c_int(cs.CUSPARSE_CSR2CSC_ALG1))
    size = C.c_size_t()
    assert R.cusparseCsr2cscEx2_bufferSize(h, *args, C.byref(size)) == 0
    cbuf = torch.empty(max(size.value, 16), dtype=torch.uint8, device=DEV)
    closed = lambda: R.cusparseCsr2cscEx2(h, *args, ptr(cbuf))  # noqa: E731
    assert ours() == 0 and closed() == 0
    torch.cuda.synchronize()
    equal = all(same(a, b) for a, b in zip(outs[0], outs[1]))
    t_ours, t_closed = timeit(ours), timeit(closed)
    nbytes = 4 * (m + 1) + 4 * nnz + width * nnz + 4 * (n + 1) + 4 * nnz + width * nnz
    return dict(op="csr2csc", case=name, values="symbolic" if dt is None else str(dt)[6:], us=t_ours * 1e6, us_closed=t_closed * 1e6,
                speedup=t_closed / t_ours, bytes=nbytes, gbs=nbytes / t_ours / 1e9, gbs_closed=nbytes / t_closed / 1e9, equal=equal,
                buffer_bytes=dict(ours=wsb, closed=size.value),
                routed=bool(L.b200conv_route(CSR2CSC, m, n, nnz, width, cs.CUSPARSE_CSR2CSC_ALG1, ptr(ws))))


def coo_orders(m, off, col):
    rows = torch.repeat_interleave(torch.arange(m, device=DEV, dtype=torch.int32), (off[1:] - off[:-1]).long())
    by_col = torch.sort(col.long() * (m + 1) + rows.long(), stable=True).indices
    g = torch.Generator(device=DEV).manual_seed(11)
    shuffle = torch.randperm(rows.numel(), device=DEV, generator=g)
    yield "row_order", rows, col
    yield "col_order", rows[by_col].contiguous(), col[by_col].contiguous()
    yield "shuffled", rows[shuffle].contiguous(), col[shuffle].contiguous()


def coosort_case(L, R, h, name, m, n, order, rows0, cols0, by_row):
    nnz = rows0.numel()
    P0 = torch.arange(nnz, device=DEV, dtype=torch.int32)
    bufs = [(torch.empty_like(rows0), torch.empty_like(cols0), torch.empty_like(P0)) for _ in range(2)]
    wsb = L.b200coosort_workspace_bytes(m, n, nnz)
    ws = torch.empty(wsb, dtype=torch.uint8, device=DEV)
    size = C.c_size_t()
    assert R.cusparseXcoosort_bufferSizeExt(h, m, n, nnz, ptr(rows0), ptr(cols0), C.byref(size)) == 0
    cbuf = torch.empty(max(size.value, 16), dtype=torch.uint8, device=DEV)
    st = torch.cuda.current_stream().cuda_stream
    sort_closed = R.cusparseXcoosortByRow if by_row else R.cusparseXcoosortByColumn

    def restore(b):
        b[0].copy_(rows0); b[1].copy_(cols0); b[2].copy_(P0)

    def ours():
        b = bufs[0]
        restore(b)
        return L.b200coosort(st, int(by_row), m, n, nnz, ptr(b[0]), ptr(b[1]), ptr(b[2]), ptr(ws), wsb)

    def closed():
        b = bufs[1]
        restore(b)
        return sort_closed(h, m, n, nnz, ptr(b[0]), ptr(b[1]), ptr(b[2]), ptr(cbuf))
    assert ours() == 0 and closed() == 0
    torch.cuda.synchronize()
    equal = all(same(a, b) for a, b in zip(bufs[0], bufs[1]))
    t_copy = timeit(lambda: restore(bufs[0]))
    t_ours, t_closed = max(timeit(ours) - t_copy, 1e-9), max(timeit(closed) - t_copy, 1e-9)
    nbytes = 24 * nnz
    op = COOSORT_ROW if by_row else COOSORT_COL
    return dict(op="coosort_by_row" if by_row else "coosort_by_col", case=name, order=order, us=t_ours * 1e6, us_closed=t_closed * 1e6,
                speedup=t_closed / t_ours, bytes=nbytes, gbs=nbytes / t_ours / 1e9, gbs_closed=nbytes / t_closed / 1e9, equal=equal,
                buffer_bytes=dict(ours=wsb, closed=size.value), routed=bool(L.b200conv_route(op, m, n, nnz, 0, 0, ptr(ws))))


def coo2csr_cases(L, R, h, name, m, off):
    nnz = int(off[-1].item())
    rows = torch.repeat_interleave(torch.arange(m, device=DEV, dtype=torch.int32), (off[1:] - off[:-1]).long())
    st = torch.cuda.current_stream().cuda_stream
    o = [torch.empty(m + 1, dtype=torch.int32, device=DEV) for _ in range(2)]
    r = [torch.empty(nnz, dtype=torch.int32, device=DEV) for _ in range(2)]
    out = []
    for op, ours, closed, res, nbytes in (
            (COO2CSR, lambda: L.b200coo2csr(st, ptr(rows), nnz, m, ptr(o[0]), 0),
             lambda: R.cusparseXcoo2csr(h, ptr(rows), nnz, m, ptr(o[1]), 0), o, 4 * nnz + 4 * (m + 1)),
            (CSR2COO, lambda: L.b200csr2coo(st, ptr(off), nnz, m, ptr(r[0]), 0),
             lambda: R.cusparseXcsr2coo(h, ptr(off), nnz, m, ptr(r[1]), 0), r, 4 * nnz + 4 * (m + 1))):
        assert ours() == 0 and closed() == 0
        torch.cuda.synchronize()
        t_ours, t_closed = timeit(ours), timeit(closed)
        out.append(dict(op="coo2csr" if op == COO2CSR else "csr2coo", case=name, us=t_ours * 1e6, us_closed=t_closed * 1e6,
                        speedup=t_closed / t_ours, bytes=nbytes, gbs=nbytes / t_ours / 1e9, gbs_closed=nbytes / t_closed / 1e9,
                        equal=same(res[0], res[1]), routed=bool(L.b200conv_route(op, m, 0, nnz, 0, 0, None))))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--quick", action="store_true")
    ap.add_argument("--json")
    ap.add_argument("--matrices", default=",".join(MATRICES))
    a = ap.parse_args()
    L = _lib.shim()
    api = cs.Api("cusparse")
    R = api.real
    h = api.cusparseCreate()
    print(f"card: {card()}", flush=True)
    out = []

    def emit(r):
        out.append(r)
        print(json.dumps(r), flush=True)
    for name in (MATRICES[:1] if a.quick else a.matrices.split(",")):
        m, n, off, col = matrix(name)
        for dt in VALUE_TYPES:
            emit(csr2csc_case(L, R, h, name, m, n, off, col, dt))
            torch.cuda.empty_cache()
        for order, rows0, cols0 in coo_orders(m, off, col):
            for by_row in (True, False):
                emit(coosort_case(L, R, h, name, m, n, order, rows0, cols0, by_row))
            torch.cuda.empty_cache()
        for r in coo2csr_cases(L, R, h, name, m, off):
            emit(r)
        del off, col
        torch.cuda.empty_cache()
    api.cusparseDestroy(h)
    if a.json:
        with open(a.json, "w") as f:
            json.dump({"card": card(), "rows": out}, f, indent=1)


if __name__ == "__main__":
    main()
