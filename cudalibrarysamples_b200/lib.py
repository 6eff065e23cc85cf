"""ctypes loader for libb200spmv.so (the product) and the real libcusparse.so.12 (handle management + GPU oracle).

The product path fails LOUDLY when the CUDA extension is missing: there is no CPU or library fallback here.

Every b200* entry point of our three libraries gets its argtypes / restype from the prototype in include/ (load()), so a
caller passes plain ints, data_ptr()s, None and floats, and ctypes converts them to exactly the C types the header names.
"""
from __future__ import annotations

import ctypes as C
import functools
import os
import re

from . import build as _build

INCLUDE_DIR = os.path.join(os.path.dirname(_build.PKG_DIR), "include")
_C_TYPES = {"int": C.c_int, "int32_t": C.c_int32, "int64_t": C.c_int64, "size_t": C.c_size_t, "uint64_t": C.c_uint64,
            "double": C.c_double, "void": None}
_PROTOTYPE = re.compile(r"\bB200\w*_EXPORT\s+([\w\s\*]+?)\s*\b(\w+)\s*\(([^)]*)\)\s*;")


def _c_type(decl: str, what: str):
    """The ctypes type of `decl`, a return type or a parameter with or without its name."""
    words = decl.replace("*", " * ").split()
    if "*" in words:
        return C.c_char_p if words[0:2] == ["const", "char"] else C.c_void_p
    words = [w for w in words if w != "const"]
    if not words or words[0] not in _C_TYPES or len(words) > 2:
        raise ValueError(f"{what}: no ctypes type for {decl!r}")
    return _C_TYPES[words[0]]


@functools.lru_cache(maxsize=None)
def prototypes(header: str) -> tuple:
    """(return type, name, parameters) of every function include/<header> tags B200*_EXPORT, cusparse* ones included."""
    with open(os.path.join(INCLUDE_DIR, header)) as f:
        return tuple(_PROTOTYPE.findall(re.sub(r"/\*.*?\*/|//[^\n]*", " ", f.read(), flags=re.S)))


def signatures(header: str) -> dict:
    """{name: (restype, argtypes)} of every b200* prototype in include/<header>."""
    sigs = {}
    for ret, name, params in prototypes(header):
        if name.startswith("b200"):
            params = [p.strip() for p in params.split(",")]
            sigs[name] = (_c_type(ret, name), [] if params in ([""], ["void"]) else [_c_type(p, name) for p in params])
    return sigs


def load(path: str, header: str = "b200spmv.h", mode: int = C.RTLD_LOCAL) -> C.CDLL:
    """CDLL(path) with every b200* function of include/<header> declared; a declared name the library lacks raises."""
    lib = C.CDLL(path, mode=mode)
    for name, (restype, argtypes) in signatures(header).items():
        fn = getattr(lib, name)
        fn.restype, fn.argtypes = restype, argtypes
    return lib


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


def _real_cusparse_candidates() -> tuple:
    # looked up on first use, so that importing this module (as load()'s subprocess callers do) does not import torch
    return (os.environ.get("B200SPMV_CUSPARSE", ""), _bundled_with_torch(), "/usr/local/cuda/lib64/libcusparse.so.12",
            "libcusparse.so.12")


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
        for p in _real_cusparse_candidates():
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
        _shim = load(path)
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
        _spsv = load(path, header="b200spsv.h")
    return _spsv


def gen() -> C.CDLL:
    """libb200gen.so: device-side synthetic-workload generators (bench / test plumbing, include/b200gen.h)."""
    global _gen
    if _gen is None:
        path = _build.GEN_LIB_PATH
        if not os.path.exists(path):
            raise RuntimeError(f"{path} is missing: run `python -c 'import __graft_entry__ as g; g.build()'`")
        _gen = load(path, header="b200gen.h")
    return _gen
