"""ctypes loader for libb200spmv.so (the product) and the real libcusparse.so.12 (handle management + GPU oracle).

The product path fails LOUDLY when the CUDA extension is missing: there is no CPU or library fallback here.
"""
from __future__ import annotations

import ctypes as C
import os

from . import build as _build

def _bundled_with_torch() -> str:
    """torch's own libcusparse.so.12 (nvidia-cusparse-cu12 wheel).  Inside a Python process that imported torch, the
    toolkit's libcusparse 12.9 cannot be loaded (torch already mapped an older libnvJitLink.so.12), so the closed
    library used for handles and as the GPU oracle is the one torch ships; the C sample binaries use the toolkit's."""
    try:
        import torch
        p = os.path.join(os.path.dirname(os.path.dirname(torch.__file__)), "nvidia", "cusparse", "lib", "libcusparse.so.12")
        return p if os.path.exists(p) else ""
    except Exception:
        return ""


REAL_CUSPARSE_CANDIDATES = (
    os.environ.get("B200SPMV_CUSPARSE", ""),
    _bundled_with_torch(),
    "/usr/local/cuda/lib64/libcusparse.so.12",
    "libcusparse.so.12",
)

_shim = None
_spsv = None
_gen = None
_real = None
_real_path = None


def real() -> C.CDLL:
    """The closed libcusparse.so.12: cusparseCreate/Destroy/SetStream/SetPointerMode, and the GPU oracle."""
    global _real, _real_path
    if _real is None:
        errors = []
        for p in REAL_CUSPARSE_CANDIDATES:
            if not p or ("/" in p and not os.path.exists(p)):
                continue
            try:
                _real = C.CDLL(p, mode=C.RTLD_LOCAL)
                _real_path = p
                break
            except OSError as e:
                errors.append(f"{p}: {e}")
        if _real is None:
            raise RuntimeError("real libcusparse.so.12 could not be loaded (set B200SPMV_CUSPARSE): " + "; ".join(errors))
    return _real


def real_cusparse_path() -> str:
    real()
    return _real_path


def shim(build_if_missing: bool = False) -> C.CDLL:
    """libb200spmv.so. Raises if it has not been built (run __graft_entry__.build())."""
    global _shim
    if _shim is None:
        # the shim must dlopen the very same libcusparse instance that creates the handles we pass to it
        os.environ["B200SPMV_CUSPARSE"] = real_cusparse_path()
        path = os.environ.get("B200SPMV_LIB") or _build.LIB_PATH   # B200SPMV_LIB: a tuning variant (scripts/sweep.py)
        if not os.path.exists(path):
            if build_if_missing:
                _build.build_native()
            else:
                raise RuntimeError(
                    f"{path} is missing: the CUDA extension was not built. Run `python -c 'import __graft_entry__ as g; "
                    "g.build()'` (nvcc, sm_90a). There is no CPU fallback.")
        lib = C.CDLL(path, mode=C.RTLD_LOCAL)
        lib.b200spmv_csr_workspace_bytes.restype = C.c_size_t
        lib.b200spmv_coo_workspace_bytes.restype = C.c_size_t
        lib.b200spmv_sell_workspace_bytes.restype = C.c_size_t
        lib.b200spmv_csr_plan_tiles_offset.restype = C.c_size_t
        lib.b200spmv_csr_plan_ctl_offset.restype = C.c_size_t
        lib.b200spmv_csr_plan_split_offset.restype = C.c_size_t
        lib.b200spmv_csr_num_tiles.restype = C.c_int64
        lib.b200spmv_version.restype = C.c_char_p
        lib.b200sddmm_csr_workspace_bytes.restype = C.c_size_t
        i64, vp = C.c_int64, C.c_void_p
        lib.b200spmm_bell.argtypes = [vp, C.c_int, C.c_int, i64, i64, i64, i64, i64, vp, vp, C.c_int32, vp, vp, C.c_int, vp, i64, C.c_int,
                                      vp, i64, C.c_int]
        lib.b200spmm_bell_route.argtypes = [vp, vp, vp, C.c_int, C.c_int, C.c_int, C.c_int]
        lib.b200spmm_coo.argtypes = [vp, C.c_int, C.c_int, i64, i64, i64, i64, vp, vp, vp, C.c_int32, vp, vp, C.c_int, vp, i64, C.c_int,
                                     vp, i64, C.c_int, C.c_int, i64, i64, i64, vp, C.c_size_t]
        lib.b200spmm_coo_workspace_bytes.argtypes = [C.c_int, C.c_int, i64, i64, i64, i64, C.c_int, C.c_int, i64]
        lib.b200spmm_coo_workspace_bytes.restype = C.c_size_t
        lib.b200spmm_coo_route.argtypes = [vp, vp, vp, C.c_int, C.c_int, C.c_int, C.c_int]
        lib.b200sddmm_bsr.argtypes = [vp, C.c_int, C.c_int, i64, i64, i64, i64, i64, vp, vp, vp, C.c_int32, C.c_int, vp, vp, C.c_int,
                                      vp, i64, i64, vp, i64, i64, C.c_int, i64, i64, i64, i64, i64]
        lib.b200sddmm_bsr_path.argtypes = [C.c_int, i64, vp, i64, i64, vp, i64, i64, C.c_int, i64, i64]
        lib.b200sddmm_bsr_route.argtypes = [vp, vp, vp, C.c_int, C.c_int, C.c_int]
        lib.b200spmm_bsr.argtypes = [vp, C.c_int, C.c_int, i64, i64, i64, i64, i64, vp, vp, vp, C.c_int32, C.c_int, vp, vp, C.c_int,
                                     vp, i64, i64, vp, i64, C.c_int, C.c_int, i64, i64, i64, i64, i64, vp, C.c_size_t]
        lib.b200spmm_bsr_workspace_bytes.argtypes = [C.c_int, i64, i64, i64, i64, C.c_int]
        lib.b200spmm_bsr_workspace_bytes.restype = C.c_size_t
        lib.b200spmm_bsr_path.argtypes = [C.c_int, i64, C.c_int, vp, vp, i64, i64, C.c_int, i64, i64]
        lib.b200spmm_bsr_route.argtypes = [vp, vp, vp, C.c_int, C.c_int, C.c_int, C.c_int]
        lib.b200spmm_csr16.argtypes = [vp, C.c_int, C.c_int, i64, i64, i64, i64, vp, vp, vp, C.c_int32, vp, vp, C.c_int, vp, i64, i64, vp,
                                       i64, C.c_int, vp, C.c_size_t]
        lib.b200spmm_csr16_workspace_bytes.argtypes = [i64, i64, i64, i64, i64]
        lib.b200spmm_csr16_workspace_bytes.restype = C.c_size_t
        lib.b200spmm_csr16_path.argtypes = [i64, vp, i64, i64]
        lib.b200spmm_csr16_route.argtypes = [vp, vp, vp, C.c_int, C.c_int, C.c_int, C.c_int]
        lib.b200spmm_csr_t.argtypes = [vp, C.c_int, C.c_int, i64, i64, i64, i64, vp, vp, vp, C.c_int32, vp, vp, C.c_int, vp, i64, i64, vp,
                                       i64, C.c_int, C.c_int, vp, C.c_size_t]
        lib.b200spmm_csr_t_plan.argtypes = [vp, i64, i64, i64, vp, vp, C.c_int32, vp, C.c_size_t]
        lib.b200spmm_csr_t_layout.argtypes = [C.c_int, i64, i64, i64, i64, i64, i64, vp]
        lib.b200spmm_csr_t_layout.restype = C.c_size_t
        lib.b200spmm_csr_t_workspace_bytes.argtypes = [C.c_int, i64, i64, i64, i64, i64, i64]
        lib.b200spmm_csr_t_workspace_bytes.restype = C.c_size_t
        lib.b200spmm_csr_t_route.argtypes = [vp, vp, vp, C.c_int, C.c_int, C.c_int, C.c_int, vp]
        lib.b200spmv_plan_trusted.argtypes = [vp, vp, C.c_int]
        lib.b200spmv_csr16.argtypes = [vp, C.c_int, C.c_int, i64, i64, i64, vp, vp, vp, C.c_int32, vp, vp, C.c_int, vp, vp, vp, C.c_size_t]
        lib.b200spmv_csr16_workspace_bytes.argtypes = [i64, i64]
        lib.b200spmv_csr16_workspace_bytes.restype = C.c_size_t
        lib.b200spmv_csr16_path.argtypes = [vp, vp]
        lib.b200spmv_csr16_route.argtypes = [vp, vp, vp, C.c_int, C.c_int, C.c_int]
        lib.b200spmv_route.argtypes = [C.c_int] * 9 + [i64] * 3
        lib.b200spmv_csr_z.argtypes = [vp, C.c_int, i64, i64, i64, vp, vp, vp, C.c_int32, vp, vp, C.c_int, vp, vp, vp, C.c_size_t]
        lib.b200spmv_csr_z_workspace_bytes.argtypes = [i64, i64]
        lib.b200spmv_csr_z_workspace_bytes.restype = C.c_size_t
        lib.b200spmv_csr_z_params.argtypes = [vp, vp, vp]
        lib.b200spsm_csr_workspace_bytes.argtypes = [i64, i64, C.c_int]
        lib.b200spsm_csr_workspace_bytes.restype = C.c_size_t
        lib.b200spsm_csr_layout.argtypes = [i64, i64, C.c_int, vp]
        lib.b200spsm_csr_analysis.argtypes = [vp, i64, i64, vp, vp, C.c_int32, C.c_int, C.c_int, C.c_int, vp, vp, vp]
        lib.b200spsm_csr_solve.argtypes = [vp, C.c_int, i64, i64, C.c_int, vp, vp, vp, C.c_int, i64, vp, i64, i64, vp, i64, i64, vp]
        lib.b200spsm_csr_tile.argtypes = [i64, C.c_int]
        lib.b200spsm_route.argtypes = [C.c_int] * 12 + [i64] * 4 + [C.c_int, C.c_int]
        _shim = lib
    return _shim


def spsv() -> C.CDLL:
    """libb200spsv.so, the opt-in CSR triangular solve (include/b200spsv.h). Raises if it has not been built."""
    global _spsv
    if _spsv is None:
        # like shim(): the library must dlopen the very libcusparse instance that creates the handles we pass to it
        os.environ["B200SPMV_CUSPARSE"] = real_cusparse_path()
        path = _build.SPSV_LIB_PATH
        if not os.path.exists(path):
            raise RuntimeError(f"{path} is missing: run `python -c 'import __graft_entry__ as g; g.build()'` (nvcc, sm_90a). "
                               "There is no CPU fallback.")
        lib = C.CDLL(path, mode=C.RTLD_LOCAL)
        lib.b200spsv_csr_workspace_bytes.restype = C.c_size_t
        lib.b200spsv_csr_workspace_bytes.argtypes = [C.c_int64, C.c_int64, C.c_int]
        lib.b200spsv_version.restype = C.c_char_p
        _spsv = lib
    return _spsv


def gen() -> C.CDLL:
    """libb200gen.so: device-side synthetic-workload generators (bench / test plumbing, include/b200gen.h)."""
    global _gen
    if _gen is None:
        path = _build.GEN_LIB_PATH
        if not os.path.exists(path):
            raise RuntimeError(f"{path} is missing: run `python -c 'import __graft_entry__ as g; g.build()'`")
        _gen = C.CDLL(path, mode=C.RTLD_LOCAL)
    return _gen
