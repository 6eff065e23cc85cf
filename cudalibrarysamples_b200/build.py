"""Build the native libraries in-tree with nvcc:

  libb200spmv.so  the product: sm_90a kernels + the cuSPARSE-symbol shim (include/b200spmv.h)
  libb200gen.so   bench / test plumbing: synthetic-workload generators on the device (include/b200gen.h)
  libb200spsv.so  the opt-in CSR triangular solve: sm_90a kernels + the cusparseSpSV_* shim (include/b200spsv.h); it does
                  not link against libb200spmv.so

The .so files are build products and git-ignored.  nvcc cross-compiles for sm_90a without a GPU, so this also runs
on a machine that has none.
"""
from __future__ import annotations

import os
import shutil
import subprocess
import sys

PKG_DIR = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(PKG_DIR, "csrc")
LIB_PATH = os.path.join(PKG_DIR, "libb200spmv.so")
GEN_LIB_PATH = os.path.join(PKG_DIR, "libb200gen.so")
SPSV_LIB_PATH = os.path.join(PKG_DIR, "libb200spsv.so")
SOURCES = ["spmv_csr.cu", "spmv_csr_flat.cu", "spmv_csr_short.cu", "spmv_csr16.cu", "spmv_csr_z.cu", "spmv_csr_transpose.cu", "spmv_coo_sell.cu", "spmv_generic.cu", "spmm_csr.cu", "spmm_coo.cu", "spmm_bell.cu", "spmm_bsr.cu", "spmm_csr16.cu", "spmm_csr_t.cu", "convert.cu", "dense_convert.cu", "batched_banded.cu", "ilu0_csr.cu", "spgemm_csr.cu", "sddmm_csr.cu", "sddmm_bsr.cu", "spsm_csr.cu", "cg_fused.cu", "bicgstab_fused.cu", "peer_sync.cu", "config.cpp", "cusparse_shim.cpp", "real_cusparse.cpp"]
GEN_SOURCES = ["workload_gen.cu"]
SPSV_SOURCES = ["spsv_csr.cu", "spsv_shim.cpp", "real_cusparse.cpp"]
HEADERS = ["spmv_common.cuh", "cg_reduce.cuh", "radix_sort.cuh", "csr_chunk_walk.cuh", "mma_sm90.cuh", "spsv_plan.cuh", "spmv_generic_kernels.cuh", "batched_banded.cuh", "config.h", "real_cusparse.h", os.path.join("..", "..", "include", "b200spmv.h"),
           os.path.join("..", "..", "include", "b200gen.h"), os.path.join("..", "..", "include", "b200spsv.h")]

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-lineinfo", "-O3", "-std=c++17",
    "-Xcompiler", "-fPIC", "-Xcompiler", "-fvisibility=default",
    "-Xptxas", "-v",
]


def nvcc() -> str:
    exe = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(exe):
        raise RuntimeError("nvcc not found: cannot build libb200spmv.so")
    return exe


def _stale(target: str, sources) -> bool:
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    deps = [os.path.join(CSRC, s) for s in list(sources) + HEADERS] + [os.path.abspath(__file__)]
    return any(os.path.exists(d) and os.path.getmtime(d) > t for d in deps)


def needs_build() -> bool:
    return _stale(LIB_PATH, SOURCES) or _stale(GEN_LIB_PATH, GEN_SOURCES) or _stale(SPSV_LIB_PATH, SPSV_SOURCES)


def _compile_and_link(sources, target, build_dir, extra_flags, log):
    os.makedirs(build_dir, exist_ok=True)
    objs = []
    procs = []
    for s in sources:
        o = os.path.join(build_dir, s + ".o")
        cmd = [nvcc(), *NVCC_FLAGS, *extra_flags, "-c", os.path.join(CSRC, s), "-o", o]
        procs.append((s, cmd, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
        objs.append(o)
    failed = None
    for s, cmd, pr in procs:                     # the translation units compile in parallel
        out, _ = pr.communicate()
        log.append("$ " + " ".join(cmd) + "\n" + out)
        if pr.returncode != 0 and failed is None:
            failed = s
    if failed:
        sys.stderr.write("\n".join(log))
        raise RuntimeError(f"nvcc failed on {failed}")
    cmd = [nvcc(), "-shared", "-gencode", "arch=compute_90a,code=sm_90a", "-o", target, *objs, "-ldl", "-lpthread"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    log.append("$ " + " ".join(cmd) + "\n" + r.stdout + r.stderr)
    if r.returncode != 0:
        sys.stderr.write(log[-1])
        raise RuntimeError("link failed")


def build_native(force: bool = False, verbose: bool = False, extra_flags=(), out_path: str | None = None,
                 tag: str = "") -> str:
    """Compile every CUDA source for sm_90a into cudalibrarysamples_b200/libb200spmv.so (+ libb200gen.so, libb200spsv.so).

    extra_flags / out_path / tag build a tuning variant of the product library (scripts/sweep.py) next to the default."""
    variant = bool(extra_flags) or out_path is not None
    log = []
    if variant:
        build_dir = os.path.join(PKG_DIR, "build", tag or "variant")
        _compile_and_link(SOURCES, out_path or LIB_PATH, build_dir, list(extra_flags), log)
        with open(os.path.join(build_dir, "build.log"), "w") as f:
            f.write("\n".join(log))
        return out_path or LIB_PATH
    build_dir = os.path.join(PKG_DIR, "build")
    if force or _stale(LIB_PATH, SOURCES):
        _compile_and_link(SOURCES, LIB_PATH, build_dir, [], log)
    if force or _stale(GEN_LIB_PATH, GEN_SOURCES):
        _compile_and_link(GEN_SOURCES, GEN_LIB_PATH, os.path.join(build_dir, "gen"), [], log)
    if force or _stale(SPSV_LIB_PATH, SPSV_SOURCES):
        _compile_and_link(SPSV_SOURCES, SPSV_LIB_PATH, os.path.join(build_dir, "spsv"), [], log)
    if log:
        with open(os.path.join(build_dir, "build.log"), "w") as f:
            f.write("\n".join(log))
        if verbose:
            print("\n".join(log))
    return LIB_PATH


if __name__ == "__main__":
    print(build_native(force="--force" in sys.argv, verbose=True))
