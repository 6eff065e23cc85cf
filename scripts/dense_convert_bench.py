#!/usr/bin/env python
"""Sparse <-> dense conversion, ours (dense_convert.cu) against the closed library on the same buffers, in one process
(DESIGN.md 3.24).

Matrices: 8192^2 and 16384^2 (and 32768^2 in fp16 only, for memory) at densities 0.1 %, 1 %, 10 % and 50 %, with uniform and
power-law row lengths (row i keeps its entries with a probability proportional to (i + 1)^-0.5, scaled to the same mean), dense
row- and column-major, fp16 / fp32 / fp64 / complex128; Blocked-ELL masks at bs 16 / 32 / 64 with half the block columns stored.
Per case:
* s2d  CSR -> dense: b200csr2dense against cusparseSparseToDense;
* d2s  dense -> CSR convert: b200dense2csr against cusparseDenseToSparse_convert, both after the closed analysis;
* bell s2d / d2s on the Blocked-ELL mask.
Each call is timed with CUDA events after a warm-up, median of three windows.  Reported per row: both times, the speed-up, GB/s of
compulsory bytes (s2d writes m n w and reads nnz (w + 4) + 4 (m + 1); the convert reads m n w and writes nnz (w + 4)) and its
share of 3.35 TB/s, bit-equality with the closed output, and b200dense_route's verdict.  The card's name and power limit are read
in the same run.
usage: python scripts/dense_convert_bench.py [--quick] [--json out.json]"""
import argparse
import ctypes as C
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from cudalibrarysamples_b200 import cusparse_api as cs  # noqa: E402
from cudalibrarysamples_b200 import lib as _lib  # noqa: E402
from scripts.sddmm_bsr_bench import card, timeit  # noqa: E402

DEV = torch.device("cuda:0")
PEAK = 3.35e12
ROW, COL = cs.CUSPARSE_ORDER_ROW, cs.CUSPARSE_ORDER_COL
VT = {torch.float16: 2, torch.float32: 0, torch.float64: 1, torch.complex128: 5}
I32 = C.c_int(cs.CUSPARSE_INDEX_32I)


def dense_matrix(m, n, density, dist, dt, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    p = torch.full((m, 1), density, device=DEV)
    if dist == "powerlaw":
        w = (torch.arange(m, device=DEV, dtype=torch.float32) + 1) ** -0.5
        p = (density * w / w.mean()).clamp(max=1.0).view(m, 1)
    mask = torch.rand(m, n, device=DEV, generator=g) < p
    v = torch.randint(1, 1 << 10, (m, n * (2 if dt.is_complex else 1)), device=DEV, generator=g, dtype=torch.int32)
    v = v.double().view(torch.complex128) if dt.is_complex else v.to(dt)
    return torch.where(mask, v, torch.zeros((), dtype=dt, device=DEV))


def call(R, name, *args):
    st = getattr(R, name)(*args)
    if st != 0:
        raise RuntimeError(f"{name}: {st}")


def csr_case(L, R, h, m, n, density, dist, dt, order):
    """(our s2d time, closed s2d time, s2d equal, our d2s time, closed d2s time, d2s equal, nnz)"""
    A = dense_matrix(m, n, density, dist, dt, 1)
    D = (A if order == ROW else A.t()).contiguous().reshape(-1)
    del A
    ld = n if order == ROW else m
    vt = VT[dt]
    w = D.element_size()
    st = torch.cuda.current_stream().cuda_stream
    dn = C.c_void_p()
    call(R, "cusparseCreateDnMat", C.byref(dn), C.c_int64(m), C.c_int64(n), C.c_int64(ld), C.c_void_p(D.data_ptr()), C.c_int(vt), C.c_int(order))
    off = torch.empty(m + 1, dtype=torch.int32, device=DEV)
    sp = C.c_void_p()
    call(R, "cusparseCreateCsr", C.byref(sp), C.c_int64(m), C.c_int64(n), C.c_int64(0), C.c_void_p(off.data_ptr()), None, None, I32, I32,
         C.c_int(0), C.c_int(vt))
    size = C.c_size_t()
    call(R, "cusparseDenseToSparse_bufferSize", h, dn, sp, 0, C.byref(size))
    buf = torch.empty(max(size.value, 16), dtype=torch.uint8, device=DEV)
    call(R, "cusparseDenseToSparse_analysis", h, dn, sp, 0, C.c_void_p(buf.data_ptr()))
    r_, c_, z = C.c_int64(), C.c_int64(), C.c_int64()
    call(R, "cusparseSpMatGetSize", sp, C.byref(r_), C.byref(c_), C.byref(z))
    nnz = z.value
    ind = [torch.empty(max(nnz, 1), dtype=torch.int32, device=DEV) for _ in range(2)]
    val = [torch.empty(max(nnz, 1), dtype=dt, device=DEV) for _ in range(2)]
    call(R, "cusparseCsrSetPointers", sp, C.c_void_p(off.data_ptr()), C.c_void_p(ind[1].data_ptr()), C.c_void_p(val[1].data_ptr()))
    closed_d2s = lambda: call(R, "cusparseDenseToSparse_convert", h, dn, sp, 0, C.c_void_p(buf.data_ptr()))  # noqa: E731
    ours_d2s = lambda: L.b200dense2csr(st, 0, m, n, nnz, D.data_ptr(), ld, order, vt, off.data_ptr(), ind[0].data_ptr(),  # noqa: E731
                                       val[0].data_ptr(), 0)
    t_cd, t_od = timeit(closed_d2s), timeit(ours_d2s)
    eq_d = torch.equal(ind[0], ind[1]) and torch.equal(val[0].view(torch.uint8), val[1].view(torch.uint8))
    if not eq_d and os.environ.get("DENSE_BENCH_DEBUG"):
        bad = (ind[0] != ind[1]).nonzero()
        k = int(bad[0]) if len(bad) else -1
        print("  mismatch: ind", len(bad), "first", k, ind[0][max(k - 3, 0):k + 3].tolist(), ind[1][max(k - 3, 0):k + 3].tolist(),
              "off", off[:4].tolist(), "val bytes equal", torch.equal(val[0].view(torch.uint8), val[1].view(torch.uint8)))
    # CSR -> dense on the converted arrays, into two fresh dense buffers
    out = [torch.empty_like(D) for _ in range(2)]
    dn2 = C.c_void_p()
    call(R, "cusparseCreateDnMat", C.byref(dn2), C.c_int64(m), C.c_int64(n), C.c_int64(ld), C.c_void_p(out[1].data_ptr()), C.c_int(vt),
         C.c_int(order))
    call(R, "cusparseSparseToDense_bufferSize", h, sp, dn2, 0, C.byref(size))
    buf2 = torch.empty(max(size.value, 16), dtype=torch.uint8, device=DEV)
    closed_s2d = lambda: call(R, "cusparseSparseToDense", h, sp, dn2, 0, C.c_void_p(buf2.data_ptr()))  # noqa: E731
    ours_s2d = lambda: L.b200csr2dense(st, 0, m, n, nnz, off.data_ptr(), ind[1].data_ptr(), val[1].data_ptr(), w, 0,  # noqa: E731
                                       out[0].data_ptr(), ld, order)
    t_cs, t_os = timeit(closed_s2d), timeit(ours_s2d)
    eq_s = torch.equal(out[0].view(torch.uint8), out[1].view(torch.uint8))
    for d in (dn, dn2):
        R.cusparseDestroyDnMat(d)
    R.cusparseDestroySpMat(sp)
    return t_os, t_cs, eq_s, t_od, t_cd, eq_d, nnz


def bell_case(L, R, h, m, bs, dt, order):
    nb = m // bs
    g = torch.Generator(device=DEV).manual_seed(bs)
    slots = nb // 2
    colind = torch.stack([torch.randperm(nb, device=DEV, generator=g)[:slots].sort().values for _ in range(nb)]).int().contiguous()
    A = dense_matrix(m, m, 0.5, "uniform", dt, 2)
    D = (A if order == ROW else A.t()).contiguous().reshape(-1)
    del A
    vt, w = VT[dt], D.element_size()
    st = torch.cuda.current_stream().cuda_stream
    ev = [torch.full((m * slots * bs * w,), 0xFF, dtype=torch.uint8, device=DEV).view(dt) for _ in range(2)]   # NaN in the -1 slots
    dn, sp = C.c_void_p(), C.c_void_p()
    call(R, "cusparseCreateDnMat", C.byref(dn), C.c_int64(m), C.c_int64(m), C.c_int64(m), C.c_void_p(D.data_ptr()), C.c_int(vt), C.c_int(order))
    call(R, "cusparseCreateBlockedEll", C.byref(sp), C.c_int64(m), C.c_int64(m), C.c_int64(bs), C.c_int64(slots * bs),
         C.c_void_p(colind.data_ptr()), C.c_void_p(ev[1].data_ptr()), I32, C.c_int(0), C.c_int(vt))
    size = C.c_size_t()
    call(R, "cusparseDenseToSparse_bufferSize", h, dn, sp, 0, C.byref(size))
    buf = torch.empty(max(size.value, 16), dtype=torch.uint8, device=DEV)
    call(R, "cusparseDenseToSparse_analysis", h, dn, sp, 0, C.c_void_p(buf.data_ptr()))
    t_cd = timeit(lambda: call(R, "cusparseDenseToSparse_convert", h, dn, sp, 0, C.c_void_p(buf.data_ptr())))
    t_od = timeit(lambda: L.b200dense2bell(st, m, m, bs, slots * bs, D.data_ptr(), m, order, w, colind.data_ptr(), ev[0].data_ptr(), 0))
    eq_d = torch.equal(ev[0].view(torch.uint8), ev[1].view(torch.uint8))
    out = [torch.empty_like(D) for _ in range(2)]
    dn2 = C.c_void_p()
    call(R, "cusparseCreateDnMat", C.byref(dn2), C.c_int64(m), C.c_int64(m), C.c_int64(m), C.c_void_p(out[1].data_ptr()), C.c_int(vt),
         C.c_int(order))
    supported = R.cusparseSparseToDense_bufferSize(h, sp, dn2, 0, C.byref(size)) == 0     # the closed library refuses Blocked-ELL
    buf2 = torch.empty(max(size.value, 16), dtype=torch.uint8, device=DEV)
    t_cs = timeit(lambda: call(R, "cusparseSparseToDense", h, sp, dn2, 0, C.c_void_p(buf2.data_ptr()))) if supported else float("nan")
    t_os = timeit(lambda: L.b200bell2dense(st, m, m, bs, slots * bs, colind.data_ptr(), ev[1].data_ptr(), w, 0, out[0].data_ptr(), m, order))
    eq_s = torch.equal(out[0].view(torch.uint8), out[1].view(torch.uint8)) if supported else None
    for d in (dn, dn2):
        R.cusparseDestroyDnMat(d)
    R.cusparseDestroySpMat(sp)
    return t_os, t_cs, eq_s, t_od, t_cd, eq_d, m * slots * bs


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--quick", action="store_true")
    ap.add_argument("--only", choices=("csr", "bell"))
    ap.add_argument("--json")
    a = ap.parse_args()
    L, R = _lib.shim(), _lib.real()
    h = C.c_void_p()
    call(R, "cusparseCreate", C.byref(h))
    call(R, "cusparseSetStream", h, C.c_void_p(torch.cuda.current_stream().cuda_stream))
    print(f"# card: {card()}")
    rows = []
    sizes = ((8192, (torch.float16, torch.float32, torch.float64, torch.complex128)), (16384, (torch.float16, torch.float32, torch.float64,
             torch.complex128)), (32768, (torch.float16,)))
    if a.quick:
        sizes = ((8192, (torch.float16, torch.float32)),)
    hdr = f"{'case':58s} {'dir':>4s} {'ours ms':>9s} {'closed ms':>9s} {'speed-up':>8s} {'GB/s':>7s} {'%peak':>6s} {'equal':>5s} {'route':>5s}"
    print(hdr)

    def report(case, direction, t_o, t_c, eq, byts, rt):
        gbs = byts / t_o / 1e9
        print(f"{case:58s} {direction:>4s} {t_o * 1e3:9.3f} {t_c * 1e3:9.3f} {t_c / t_o:8.2f} {gbs:7.0f} {100 * byts / t_o / PEAK:6.1f} "
              f"{str(eq):>5s} {rt:5d}", flush=True)
        rows.append(dict(case=case, dir=direction, ours_s=t_o, closed_s=t_c, speedup=t_c / t_o, gbs=gbs, equal=eq, route=rt))

    for m, dts in (() if a.only == "bell" else sizes):
        for dt in dts:
            for order in (ROW, COL):
                for dist in ("uniform", "powerlaw"):
                    for dens in ((0.01, 0.1) if a.quick else (0.001, 0.01, 0.1, 0.5)):
                        t_os, t_cs, eq_s, t_od, t_cd, eq_d, nnz = csr_case(L, R, h, m, m, dens, dist, dt, order)
                        w = torch.empty(0, dtype=dt).element_size()
                        case = f"csr {m}^2 {str(dt)[6:]} {'row' if order == ROW else 'col'} {dist} {dens:g}"
                        report(case, "s2d", t_os, t_cs, eq_s, m * m * w + nnz * (w + 4) + 4 * (m + 1),
                               L.b200dense_route(0, 1, order, VT[dt], 2, 2, 0, m, m, nnz, 1, 0, 0))
                        report(case, "d2s", t_od, t_cd, eq_d, m * m * w + nnz * (w + 4),
                               L.b200dense_route(1, 1, order, VT[dt], 2, 2, 0, m, m, nnz, 1, 0, 0))
                        torch.cuda.empty_cache()
    for m in (() if a.only == "csr" else (4096,) if a.quick else (8192, 16384)):
        for bs in (16, 32, 64):
            for dt in (torch.float16, torch.float32):
                for order in (ROW, COL):
                    t_os, t_cs, eq_s, t_od, t_cd, eq_d, stored = bell_case(L, R, h, m, bs, dt, order)
                    w = torch.empty(0, dtype=dt).element_size()
                    case = f"bell {m}^2 bs{bs} {str(dt)[6:]} {'row' if order == ROW else 'col'}"
                    report(case, "s2d", t_os, t_cs, eq_s, m * m * w + stored * w + stored // (bs * bs) * 4,
                           L.b200dense_route(0, 5, order, VT[dt], 2, 2, 0, m, m, stored, 1, 0, bs))
                    report(case, "d2s", t_od, t_cd, eq_d, stored * w * 2, L.b200dense_route(1, 5, order, VT[dt], 2, 2, 0, m, m, stored, 1, 0, bs))
                    torch.cuda.empty_cache()
    R.cusparseDestroy(h)
    if a.json:
        with open(a.json, "w") as f:
            json.dump(dict(card=card(), rows=rows), f, indent=1)


if __name__ == "__main__":
    main()
