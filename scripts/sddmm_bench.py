"""Times cusparseSDDMM of libb200spmv.so against the closed libcusparse on one GPU and prints one JSON line.

Cases (C's pattern from cudalibrarysamples_b200.workloads, values uniform, alpha 1, beta 0):
  rmat_*     R-MAT 1M x 1M, 16 per row.  A is M x K row-major, B an N x K row-major feature matrix with opB = TRANSPOSE: both
             operands K-contiguous, the GNN / attention layout.  fp32 at K = 32, 64, 128 and fp64 at K = 64.
  sample_*   the same pattern in the sddmm_csr sample's layout (B K x N row-major, NON_TRANSPOSE), fp32, K = 64: ours with the
             buffer cusparseSDDMM_bufferSize asks for (B copied K-contiguous per call) and with a NULL buffer (strided loads).
  stencil_*  the 5-point 2048^2 pattern (high locality), K-contiguous layout, fp32, K = 64.
Ours is timed through b200sddmm_csr, so every case measures the kernel even where the route of cusparseSDDMM forwards it; the
closed library through its own cusparseSDDMM.  Each call is timed with CUDA events over --reps back-to-back calls after --warmup calls.  Reported per case: us per call, GFLOP/s
(2 nnz K flop), effective GB/s on the compulsory bytes (offsets + nnz (4 + size) + M K size + K N size at beta = 0), which bound
applies at the data-sheet rates of an H100 SXM (3.35 TB/s; 67 TFLOP/s fp32, 34 fp64), and the largest error of each side against an
fp64 reference, as a multiple of the dot-product error bound K u sum|a||b|.  The card name and power limit are queried in the same
run.

    python scripts/sddmm_bench.py [--reps 20] [--warmup 5] [--rows 1048576]
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

from cudalibrarysamples_b200 import cusparse_api as cs  # noqa: E402
from cudalibrarysamples_b200 import lib as _lib  # noqa: E402
from cudalibrarysamples_b200 import workloads as W  # noqa: E402

NT, TR = cs.CUSPARSE_OPERATION_NON_TRANSPOSE, cs.CUSPARSE_OPERATION_TRANSPOSE
ROW = cs.CUSPARSE_ORDER_ROW
PEAK_BW = 3.35e12
PEAK_FLOPS = {torch.float32: 67e12, torch.float64: 34e12}


def card():
    name = torch.cuda.get_device_name(0)
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                            capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:
        pl = ""
    return name, pl


def run_ours(m, n, k, off, col, A, B, dtype, opB, buffer, reps, warmup):
    """us per b200sddmm_csr call (the kernel itself, whatever the route of cusparseSDDMM decides) and the C it computes"""
    lib = _lib.shim()
    val = torch.zeros(col.numel(), dtype=dtype, device="cuda")
    dt = int(dtype == torch.float64)
    sbk, sbj = (1, k) if opB == TR else (n, 1)
    i64 = C.c_int64
    size = lib.b200sddmm_csr_workspace_bytes(dt, i64(m), i64(n), i64(k), i64(k), i64(1), i64(sbk), i64(sbj), 1, i64(0), i64(0))
    buf = torch.empty(max(size, 16), dtype=torch.uint8, device="cuda") if buffer else None
    one, zero = cs._CT[dtype](1.0), cs._CT[dtype](0.0)
    fn = lib.b200sddmm_csr
    argv = (C.c_void_p(torch.cuda.current_stream().cuda_stream), dt, i64(m), i64(n), i64(k), i64(col.numel()), C.c_void_p(off.data_ptr()),
            C.c_void_p(col.data_ptr()), C.c_void_p(val.data_ptr()), 0, C.byref(one), C.byref(zero), 0, C.c_void_p(A.data_ptr()), i64(k),
            i64(1), C.c_void_p(B.data_ptr()), i64(sbk), i64(sbj), 1, i64(0), i64(0), i64(0), i64(0),
            C.c_void_p(0 if buf is None else buf.data_ptr()), C.c_size_t(size if buffer else 0))
    for _ in range(warmup):
        assert fn(*argv) == 0
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn(*argv)
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps * 1e3, val, size


def run(impl, m, n, k, off, col, A, B, dtype, opB, buffer, reps, warmup):
    """us per cusparseSDDMM call and the C it computes (beta = 0, so every call writes the same values)"""
    api = cs.Api(impl)
    val = torch.zeros(col.numel(), dtype=dtype, device="cuda")
    h = api.cusparseCreate()
    br, bc = (k, n) if opB == NT else (n, k)
    matA = api.cusparseCreateDnMat(m, k, k, A, ROW)
    matB = api.cusparseCreateDnMat(br, bc, bc, B, ROW)
    matC = api.cusparseCreateCsr(m, n, col.numel(), off, col, val)
    ct = cs._VT[dtype]
    size = api.cusparseSDDMM_bufferSize(h, NT, opB, 1.0, matA, matB, 0.0, matC, ct)
    buf = torch.empty(max(size, 16), dtype=torch.uint8, device="cuda") if buffer else None
    api.cusparseSDDMM_preprocess(h, NT, opB, 1.0, matA, matB, 0.0, matC, ct, cs.CUSPARSE_SDDMM_ALG_DEFAULT, buf)
    one, zero = cs._CT[dtype](1.0), cs._CT[dtype](0.0)
    fn = api.lib.cusparseSDDMM
    argv = (h, C.c_int(NT), C.c_int(opB), C.cast(C.pointer(one), C.c_void_p), matA, matB, C.cast(C.pointer(zero), C.c_void_p), matC,
            C.c_int(ct), C.c_int(cs.CUSPARSE_SDDMM_ALG_DEFAULT), C.c_void_p(0 if buf is None else buf.data_ptr()))
    for _ in range(warmup):
        assert fn(*argv) == 0
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn(*argv)
    b.record()
    torch.cuda.synchronize()
    api.cusparseDestroyDnMat(matA)
    api.cusparseDestroyDnMat(matB)
    api.cusparseDestroySpMat(matC)
    api.cusparseDestroy(h)
    return a.elapsed_time(b) / reps * 1e3, val, size


def ref_error(off, col, A, Bt, out, k, dtype):
    """max |out - ref| / (K u sum|a||b|) over all entries, ref and sum|a||b| in fp64 (chunks of 1M entries)"""
    m = off.numel() - 1
    rows = torch.repeat_interleave(torch.arange(m, device="cuda"), (off[1:] - off[:-1]).long())
    u = torch.finfo(dtype).eps / 2
    worst = 0.0
    A64, B64 = A.view(m, k).double(), Bt.double()
    for s in range(0, col.numel(), 1 << 20):
        r, c = rows[s:s + (1 << 20)], col[s:s + (1 << 20)].long()
        pa, pb = A64[r], B64[c]
        ref = (pa * pb).sum(1)
        bound = k * u * (pa.abs() * pb.abs()).sum(1)
        err = (out[s:s + (1 << 20)].double() - ref).abs()
        worst = max(worst, float((err / bound.clamp_min(1e-300)).max()))
    return worst


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rows", type=int, default=1 << 20)
    args = ap.parse_args()
    name, pl = card()
    torch.manual_seed(0)
    rm = W.rmat_csr(args.rows, avg_nnz=16, seed=42, val_seed=43)
    st = W.stencil5_csr(2048)
    cases = []
    plan = [("rmat_f32_k32", rm, torch.float32, 32, TR, True), ("rmat_f32_k64", rm, torch.float32, 64, TR, True),
            ("rmat_f32_k128", rm, torch.float32, 128, TR, True), ("rmat_f64_k64", rm, torch.float64, 64, TR, True),
            ("sample_f32_k64_copy", rm, torch.float32, 64, NT, True), ("sample_f32_k64_strided", rm, torch.float32, 64, NT, False),
            ("stencil_f32_k64", st, torch.float32, 64, TR, True)]
    for label, (off, col, _), dtype, k, opB, buffer in plan:
        m = n = off.numel() - 1
        nnz = col.numel()
        A = torch.rand(m * k, dtype=dtype, device="cuda") - 0.5
        Bt = torch.rand(n, k, dtype=dtype, device="cuda") - 0.5          # op(B)^T: row j = column j of op(B)
        B = Bt.reshape(-1) if opB == TR else Bt.t().contiguous().reshape(-1)
        us, out, size = run_ours(m, n, k, off, col, A, B, dtype, opB, buffer, args.reps, args.warmup)
        err = ref_error(off, col, A, Bt, out, k, dtype)
        del out
        try:
            us_ref, out_ref, _ = run("cusparse", m, n, k, off, col, A, B, dtype, opB, True, args.reps, args.warmup)
            err_ref = ref_error(off, col, A, Bt, out_ref, k, dtype)
            del out_ref
        except cs.CuSparseError as e:
            us_ref, err_ref = None, str(e)
        vsz = torch.finfo(dtype).bits // 8
        flops = 2.0 * nnz * k
        bytes_ = (m + 1) * 4 + nnz * (4 + vsz) + m * k * vsz + k * n * vsz
        t_bw, t_fl = bytes_ / PEAK_BW, flops / PEAK_FLOPS[dtype]
        cases.append(dict(case=label, m=m, n=n, k=k, nnz=nnz, buffer_bytes=size if buffer else 0, us_b200=round(us, 2),
                          us_cusparse=None if us_ref is None else round(us_ref, 2),
                          speedup=None if us_ref is None else round(us_ref / us, 3), gflops_b200=round(flops / us / 1e3, 1),
                          gbs_b200=round(bytes_ / us / 1e3, 1), bound="memory" if t_bw >= t_fl else "compute",
                          floor_us=round(max(t_bw, t_fl) * 1e6, 2), err_over_bound_b200=err, err_over_bound_cusparse=err_ref))
        print(f"{label:24s} ours {us:9.1f} us  cusparse {us_ref if us_ref is None else round(us_ref, 1)} us  "
              f"err/bound {err:.3g} / {err_ref}", file=sys.stderr, flush=True)
        del A, B, Bt
        torch.cuda.empty_cache()
    print(json.dumps(dict(bench="sddmm_csr", gpu=name, power_limit_w=pl, reps=args.reps, warmup=args.warmup, cases=cases)))


if __name__ == "__main__":
    main()
