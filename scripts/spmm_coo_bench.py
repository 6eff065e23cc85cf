#!/usr/bin/env python
"""COO SpMM, ours (b200spmm_coo) against the closed library's cusparseSpMM on the same buffers, in one process (DESIGN.md 3.15).

Matrices: R-MAT 1M x 1M (16 per row, workloads.rmat_csr), uniform 32 per row (512K x 512K, seeded), the 7-point Laplacian on a 100^3
grid (workloads.laplace7_csr), and the samples' 4 x 4.  Per case: fp32 / fp64, N, B and C both column-major or both row-major, opA
N / T.  Ours and the closed library alternate case by case; each side runs as a CUDA graph of --calls products, timed with CUDA events
after a warm-up, median of --reps replays.  For opA = N the CSR kernel (b200spmm_csr_ws) runs on the same matrix with CSR offsets, to
show what the non-zero split buys over one warp per row.  `diff` is max |ours - closed| / max |closed|.  --unsorted records what the
closed library returns for a COO A whose entries are not row-sorted, against an fp64 product.  The card's name and power limit are read
in the same run.
usage: python scripts/spmm_coo_bench.py [--quick | --sweep | --unsorted | --batched] [--json out.json]"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from cudalibrarysamples_b200 import cusparse_api as cs  # noqa: E402
from cudalibrarysamples_b200 import lib as _lib  # noqa: E402
from cudalibrarysamples_b200 import workloads as W  # noqa: E402

DEV = torch.device("cuda:0")
ROW, COL = cs.CUSPARSE_ORDER_ROW, cs.CUSPARSE_ORDER_COL
NT, TR = cs.CUSPARSE_OPERATION_NON_TRANSPOSE, cs.CUSPARSE_OPERATION_TRANSPOSE


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name(0)


def matrix(name, dt):
    """(rows, cols, off, row, col, val) on the device, row-sorted"""
    if name == "rmat":
        off, col, val = W.rmat_csr(1 << 20, avg_nnz=16, seed=42, val_seed=43, dtype=dt)
        rows = 1 << 20
    elif name == "uniform":
        rows = 1 << 19
        g = torch.Generator(device=DEV).manual_seed(5)
        col = torch.randint(0, rows, (rows * 32,), device=DEV, generator=g, dtype=torch.int32)
        col = col.view(rows, 32).sort(dim=1).values.reshape(-1).contiguous()
        off = torch.arange(0, rows * 32 + 1, 32, device=DEV, dtype=torch.int32)
        val = (torch.rand(rows * 32, device=DEV, generator=g, dtype=torch.float64) * 2 - 1).to(dt)
    elif name == "laplace7":
        off, col, val = W.laplace7_csr(100, dtype=dt)
        rows = 100 ** 3
    else:                                                     # the samples' 4 x 4
        from oracle import oracle as O
        T = O.TOY
        rows = 4
        off, col = torch.tensor(T["csr_off"], device=DEV), torch.tensor(T["csr_col"], device=DEV)
        val = torch.tensor(T["val"], device=DEV).to(dt)
    return rows, rows, off, W.csr_to_coo_rows(off), col, val


def graph_time(fn, calls, reps, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    try:
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        g = torch.cuda.CUDAGraph()
        with torch.cuda.stream(s):
            with torch.cuda.graph(g, stream=s):
                for _ in range(calls):
                    fn()
        torch.cuda.synchronize()
        g.replay()
        torch.cuda.synchronize()
        launch = lambda: g.replay()          # noqa: E731
    except RuntimeError:                     # not capturable: the same loop, launched eagerly
        torch.cuda.synchronize()

        def launch():
            for _ in range(calls):
                fn()
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        launch()
        b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b) * 1e3 / calls)
    return float(np.median(ts))


class Closed:
    """cusparseSpMM of the closed library on a COO descriptor over the caller's buffers"""

    def __init__(self, rows, cols, row, col, val, n, Bs, ldb, Cs, ldc, order, op, alg=cs.CUSPARSE_SPMM_ALG_DEFAULT, batches=1,
                 a_stride=0, b_stride=0, c_stride=0):
        self.api = api = cs.Api("cusparse")
        self.h = api.cusparseCreate()
        self.ct = cs._VT[val.dtype]
        nnz = row.numel() // batches
        self.matA = api.cusparseCreateCoo(rows, cols, nnz, row, col, val)
        if batches > 1:
            api._call(api.real, "cusparseCooSetStridedBatch", self.matA, C.c_int(batches), C.c_int64(a_stride))
        kr, cr = (cols, rows) if op == NT else (rows, cols)
        self.matB = api.cusparseCreateDnMat(kr, n, ldb, Bs, order)
        self.matC = api.cusparseCreateDnMat(cr, n, ldc, Cs, order)
        if batches > 1:
            if b_stride:
                api.cusparseDnMatSetStridedBatch(self.matB, batches, b_stride)
            api.cusparseDnMatSetStridedBatch(self.matC, batches, c_stride)
        self.op, self.alg = op, alg
        size = api.cusparseSpMM_bufferSize(self.h, op, NT, 1.0, self.matA, self.matB, 0.0, self.matC, self.ct, alg)
        self.buf = torch.empty(max(size, 16), dtype=torch.uint8, device=DEV)
        api.cusparseSpMM_preprocess(self.h, op, NT, 1.0, self.matA, self.matB, 0.0, self.matC, self.ct, alg, self.buf)
        sc = cs._CT[val.dtype]
        self.a1, self.b0 = sc(1.0), sc(0.0)

    def __call__(self):
        self.api.cusparseSetStream(self.h, torch.cuda.current_stream().cuda_stream)
        st = self.api.real.cusparseSpMM(self.h, self.op, NT, C.byref(self.a1), self.matA, self.matB, C.byref(self.b0), self.matC, self.ct,
                                        self.alg, C.c_void_p(self.buf.data_ptr()))
        assert st == 0, st

    def close(self):
        a = self.api
        a.cusparseDestroySpMat(self.matA)
        a.cusparseDestroyDnMat(self.matB)
        a.cusparseDestroyDnMat(self.matC)
        a.cusparseDestroy(self.h)


def ours_fn(rows, cols, row, col, val, n, Bs, ldb, Cs, ldc, order, op, batches=1, a_stride=0, b_stride=0, c_stride=0):
    lib = _lib.shim()
    dt = 1 if val.dtype == torch.float64 else 0
    nnz = row.numel() // batches
    ws_bytes = lib.b200spmm_coo_workspace_bytes(dt, int(op == TR), rows, cols, n, nnz, int(order == ROW), batches, b_stride)
    ws = torch.empty(max(ws_bytes, 16), dtype=torch.uint8, device=DEV)
    sc = cs._CT[val.dtype]
    a1, b0 = sc(1.0), sc(0.0)

    def fn(_keep=(ws, a1, b0)):
        rc = lib.b200spmm_coo(torch.cuda.current_stream().cuda_stream, dt, int(op == TR), rows, cols, n, nnz, row.data_ptr(), col.data_ptr(),
                              val.data_ptr(), 0, C.addressof(a1), C.addressof(b0), 0, Bs.data_ptr(), ldb, int(order == ROW), Cs.data_ptr(),
                              ldc, int(order == ROW), batches, a_stride, b_stride, c_stride, ws.data_ptr(), ws_bytes)
        assert rc == 0, rc
    return fn


def csr_fn(rows, cols, off, col, val, n, Bs, ldb, Cs, ldc, order):
    lib = _lib.shim()
    dt = 1 if val.dtype == torch.float64 else 0
    lib.b200spmm_csr_workspace_bytes.restype = C.c_size_t
    wsb = lib.b200spmm_csr_workspace_bytes(C.c_int(dt), C.c_int64(cols), C.c_int64(n), C.c_int(int(order == ROW)))
    ws = torch.empty(max(wsb, 16), dtype=torch.uint8, device=DEV)
    sc = cs._CT[val.dtype]
    a1, b0 = sc(1.0), sc(0.0)
    i64 = C.c_int64

    def fn(_keep=(ws, a1, b0)):
        rc = lib.b200spmm_csr_ws(C.c_void_p(torch.cuda.current_stream().cuda_stream), C.c_int(dt), i64(rows), i64(cols), i64(n),
                                 i64(col.numel()), C.c_void_p(off.data_ptr()), C.c_void_p(col.data_ptr()), C.c_void_p(val.data_ptr()),
                                 C.c_int32(0), C.c_void_p(C.addressof(a1)), C.c_void_p(C.addressof(b0)), C.c_int(0),
                                 C.c_void_p(Bs.data_ptr()), i64(ldb), C.c_int(int(order == ROW)), C.c_void_p(Cs.data_ptr()), i64(ldc),
                                 C.c_int(int(order == ROW)), C.c_void_p(ws.data_ptr()))
        assert rc == 0, rc
    return fn


def run_case(mat, n, order, op, calls, reps, warmup):
    rows, cols, off, row, col, val = mat
    kr, cr = (cols, rows) if op == NT else (rows, cols)
    g = torch.Generator(device=DEV).manual_seed(11)
    B = (torch.rand(kr * n, device=DEV, generator=g, dtype=torch.float64) * 2 - 1).to(val.dtype)
    ldb, ldc = (n, n) if order == ROW else (kr, cr)
    out = dict(nnz=int(row.numel()), rows=rows, n=n, order="row" if order == ROW else "col", op="N" if op == NT else "T",
               dtype="f64" if val.dtype == torch.float64 else "f32")
    Co = torch.zeros(cr * n, dtype=val.dtype, device=DEV)
    Cc = torch.zeros(cr * n, dtype=val.dtype, device=DEV)
    ours = ours_fn(rows, cols, row, col, val, n, B, ldb, Co, ldc, order, op)
    out["ours_us"] = graph_time(ours, calls, reps, warmup)
    try:
        closed = Closed(rows, cols, row, col, val, n, B, ldb, Cc, ldc, order, op)
        try:
            out["closed_us"] = graph_time(closed, calls, reps, warmup)
        finally:
            closed.close()
        out["diff"] = float((Co.double() - Cc.double()).abs().max() / Cc.double().abs().max().clamp(min=1e-300))
        out["speedup"] = out["closed_us"] / out["ours_us"]
    except (cs.CuSparseError, AssertionError) as e:
        out["closed_us"], out["diff"] = None, f"rejected: {e}"
    if op == NT:
        Cs = torch.zeros(cr * n, dtype=val.dtype, device=DEV)
        out["csr_us"] = graph_time(csr_fn(rows, cols, off, col, val, n, B, ldb, Cs, ldc, order), calls, reps, warmup)
        del Cs
    vb = val.element_size()
    out["gbs"] = (row.numel() * (8 + vb) + kr * n * vb + cr * n * vb) / out["ours_us"] / 1e3     # compulsory bytes / our time
    del B, Co, Cc
    torch.cuda.empty_cache()
    return out


def fmt(r):
    cl = f"{r['closed_us']:.1f}" if r.get("closed_us") else "rejected"
    sp = f"{r['speedup']:.2f}x" if r.get("speedup") else "-"
    csr = f"{r['csr_us']:.1f}" if r.get("csr_us") else "-"
    d = f"{r['diff']:.1e}" if isinstance(r.get("diff"), float) else str(r.get("diff"))[:30]
    return (f"| {r['matrix']} | {r['dtype']} | {r['op']} | {r['order']} | {r['n']} | {r['ours_us']:.1f} | {cl} | {sp} | {csr} | "
            f"{r['gbs']:.0f} | {d} |")


def unsorted_finding():
    """the closed library's result for a shuffled COO A (R-MAT 64K, N 32, fp64), ours on the same entries, both against fp64"""
    res = []
    for dt in (torch.float32, torch.float64):
        off, col, val = W.rmat_csr(1 << 16, avg_nnz=16, seed=3, val_seed=4, dtype=dt)
        row = W.csr_to_coo_rows(off)
        perm = torch.randperm(row.numel(), device=DEV, generator=torch.Generator(device=DEV).manual_seed(9))
        rows = 1 << 16
        n = 32
        B = (torch.rand(rows * n, device=DEV, dtype=torch.float64) * 2 - 1)
        A = torch.sparse_coo_tensor(torch.stack([row.long(), col.long()]), val.double(), (rows, rows))
        ref = (A @ B.view(n, rows).t()).t().reshape(-1)                   # column-major C
        for name, (r, c, v) in (("sorted", (row, col, val)), ("shuffled", (row[perm], col[perm], val[perm]))):
            Bd = B.to(dt)
            Cc, Co = torch.zeros(rows * n, dtype=dt, device=DEV), torch.zeros(rows * n, dtype=dt, device=DEV)
            entry = dict(dtype=str(dt).split(".")[-1], entries=name)
            try:
                cl = Closed(rows, rows, r.contiguous(), c.contiguous(), v.contiguous(), n, Bd, rows, Cc, rows, COL, NT)
                cl()
                torch.cuda.synchronize()
                cl.close()
                entry["closed_err"] = float((Cc.double() - ref).abs().max())
            except (cs.CuSparseError, AssertionError) as e:
                entry["closed_err"] = f"rejected: {e}"
            ours_fn(rows, rows, r.contiguous(), c.contiguous(), v.contiguous(), n, Bd, rows, Co, rows, COL, NT)()
            torch.cuda.synchronize()
            entry["ours_err"] = float((Co.double() - ref).abs().max())
            res.append(entry)
            print(f"| {entry['dtype']} | {name} | {entry['closed_err']} | {entry['ours_err']:.3g} |", flush=True)
    return res


def batched(calls, reps, warmup):
    """strided batch of 8 uniform 64K x 64K matrices (32 per row), N 32, column-major, fp32; A strided and A broadcast"""
    res = []
    rows, nb, n = 1 << 16, 8, 32
    g = torch.Generator(device=DEV).manual_seed(21)
    col = torch.randint(0, rows, (nb, rows, 32), device=DEV, generator=g, dtype=torch.int32).sort(dim=2).values.reshape(-1).contiguous()
    row = torch.arange(rows, device=DEV, dtype=torch.int32).repeat_interleave(32).repeat(nb).contiguous()
    val = torch.rand(nb * rows * 32, device=DEV, generator=g) * 2 - 1
    B = torch.rand(nb * rows * n, device=DEV, generator=g) * 2 - 1
    nnz = rows * 32
    for a_stride in (nnz, 0):
        Co, Cc = torch.zeros(nb * rows * n, device=DEV), torch.zeros(nb * rows * n, device=DEV)
        r = dict(matrix=f"uniform 64K x{nb} ({'A strided' if a_stride else 'A broadcast'})", dtype="f32", op="N", order="col", n=n)
        r["ours_us"] = graph_time(ours_fn(rows, rows, row, col, val, n, B, rows, Co, rows, COL, NT, nb, a_stride, rows * n, rows * n),
                                  calls, reps, warmup)
        cl = Closed(rows, rows, row, col, val, n, B, rows, Cc, rows, COL, NT, cs.CUSPARSE_SPMM_COO_ALG4, nb, a_stride, rows * n, rows * n)
        r["closed_us"] = graph_time(cl, calls, reps, warmup)
        cl.close()
        r["speedup"] = r["closed_us"] / r["ours_us"]
        r["diff"] = float((Co - Cc).abs().max() / Cc.abs().max())
        r["gbs"] = (nb * nnz * 12 + 2 * nb * rows * n * 4) / r["ours_us"] / 1e3
        res.append(r)
        print(fmt(r), flush=True)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--quick", action="store_true", help="the 4 x 4 and Laplace 7-pt at N 32 only: a rehearsal, not a measurement")
    ap.add_argument("--sweep", action="store_true", help="R-MAT only, N 32 / 128, opA N: a short run, e.g. to compare builds")
    ap.add_argument("--unsorted", action="store_true", help="only the unsorted-A finding")
    ap.add_argument("--batched", action="store_true", help="only the strided-batch cases")
    ap.add_argument("--calls", type=int, default=10)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--json", default="")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "spmm_coo_bench.py measures on the GPU; there is nothing to measure without one"
    ch, pa, fo = C.c_int32(), C.c_int32(), C.c_int64()
    _lib.shim().b200spmm_coo_params(C.byref(ch), C.byref(pa), C.byref(fo))
    res = {"card": card(), "chunk": ch.value, "lib": os.environ.get("B200SPMV_LIB", "default"), "cases": []}
    print(f"# {res['card']}  chunk={ch.value}  lib={res['lib']}")
    if a.unsorted:
        print("| dtype | entries | closed max err vs fp64 | ours max err vs fp64 |\n|---|---|---|---|")
        res["unsorted"] = unsorted_finding()
    print("| matrix | type | opA | order | N | ours us | closed us | speedup | csr us | ours GB/s | diff |")
    print("|---|---|---|---|---|---|---|---|---|---|---|")
    if a.batched:
        res["cases"] += batched(a.calls, a.reps, a.warmup)
    if not (a.unsorted or a.batched):
        mats = ["toy", "laplace7"] if a.quick else ["rmat"] if a.sweep else ["toy", "laplace7", "uniform", "rmat"]
        ns = [32] if a.quick else [32, 128] if a.sweep else [8, 32, 64, 128]
        ops = [NT] if a.sweep else [NT, TR]
        for name in mats:
            for dt in (torch.float32, torch.float64):
                mat = matrix(name, dt)
                for op in ops:
                    for order in (COL, ROW):
                        for n in ns:
                            r = run_case(mat, n, order, op, a.calls, a.reps, a.warmup)
                            r["matrix"] = name
                            res["cases"].append(r)
                            print(fmt(r), flush=True)
                del mat
                torch.cuda.empty_cache()
    if a.json:
        os.makedirs(os.path.dirname(os.path.abspath(a.json)), exist_ok=True)
        with open(a.json, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
