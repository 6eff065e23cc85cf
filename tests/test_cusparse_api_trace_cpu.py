"""CPU: the C calls every helper of cusparse_api issues, against a trace recorded in tests/golden/cusparse_api_trace.json.

The real library, the shim and libb200spsv.so are replaced by recorders that return CUSPARSE_STATUS_SUCCESS and fill the
out-parameters (descriptors, a fixed workspace size, zero-pivot positions, cusparseSpMatGetSize, the stats counters); stream
synchronisation and the timing events are recorded as well, and every tensor lives on the CPU.  Each argument is normalised:
integers by value, pointers into the case's tensors by name, tensors a helper allocated by byte size and dtype, host alpha / beta
by value read at the width of the call's compute type, a handle or descriptor by the create call that produced it.

A successful case must issue the golden calls that take a handle or do work, in the same order (synchronize and event records
included); its descriptor create / set / destroy calls must match as a multiset; every object it creates is destroyed exactly once,
after its last use; and it returns the same object.  A failing case must raise the same CuSparseError and release at least what
the golden run released.

Regenerate the golden file with `python tests/test_cusparse_api_trace_cpu.py --record tests/golden/cusparse_api_trace.json`."""
import collections
import ctypes as C
import functools
import gc
import hashlib
import json
import os
import re
import sys
import types

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from cudalibrarysamples_b200 import cusparse_api as cs  # noqa: E402
from cudalibrarysamples_b200 import lib as _lib  # noqa: E402

GOLDEN = os.path.join(ROOT, "tests", "golden", "cusparse_api_trace.json")
BUFFER_SIZE = 8             # below the 16-byte floor of the helpers' workspace allocations
STREAM = 0x5157
_BYREF = type(C.byref(C.c_int()))
# (name pattern, positions of alpha / beta, position of the compute type) of the generic-API calls
_SCALARS = ((r"cusparseSpMV(_bufferSize|_preprocess)?", (2, 5), 7),
            (r"cusparse(SpMM|SDDMM)(_bufferSize|_preprocess)?", (3, 6), 8),
            (r"cusparseSpSV_(bufferSize|analysis|solve)", (2,), 6),
            (r"cusparseSpSM_(bufferSize|analysis|solve)", (3,), 7))
_FACTORIES = ("empty", "full", "zeros", "ones", "tensor", "empty_like", "zeros_like")
# spmm_batched did not put its handle in device pointer mode for a tensor alpha; it may now do so, right after cusparseSetStream
DEVICE_MODE_ADDED = {"spmm_batched_tensor_alpha"}


def _is_descriptor_call(name):
    """Descriptor create / set / destroy calls (and the handle's destroy): compared as a multiset, not in order."""
    if name in ("cusparseCreate", "cusparseCreateIdentityPermutation"):
        return False
    return (name.startswith("cusparseCreate") or "Destroy" in name or name.endswith(("_createDescr", "_destroyDescr"))
            or re.search(r"Set(StridedBatch|Attribute|Values|Pointers|MatIndexBase|MatType)$", name) is not None)


class _Recorder:
    def __init__(self, fail=None):
        self.fail = dict(fail or {})
        self.entries = []               # (text, name, objects used, object destroyed or None)
        self.labels = {STREAM: "stream"}  # address -> label: tensors, handles, descriptors
        self.tensors = []               # (name, tensor) of the case's own tensors
        self.objects = {}               # handle value -> label of the objects created through the recorders
        self.next_object = 0x1000
        self.pivots = 0

    # ---- the case's tensors and the helpers' allocations -------------------------------------------------------------
    def t(self, name, tensor):
        self.tensors.append((name, tensor))
        self.labels[tensor.data_ptr()] = name
        return tensor

    def alloc(self, tensor):
        if isinstance(tensor, torch.Tensor) and tensor.numel():
            self.labels[tensor.data_ptr()] = f"alloc({tensor.numel() * tensor.element_size()}B,{str(tensor.dtype)[6:]})"
        return tensor

    def label(self, x):
        if isinstance(x, torch.Tensor):
            for name, t in self.tensors:
                if x is t:
                    return name
            return f"{self.labels.get(x.data_ptr(), '?tensor')}{list(x.shape)}"
        if isinstance(x, C.c_void_p):
            return self.labels.get(x.value, "NULL" if not x.value else "?ptr")
        if isinstance(x, (tuple, list)):
            return [self.label(v) for v in x]
        if isinstance(x, dict):
            return {k: self.label(v) for k, v in x.items()}
        return x

    # ---- the recorded calls --------------------------------------------------------------------------------------------
    def _arg(self, a, ct):
        if isinstance(a, _BYREF):
            o = a._obj
            return f"&{type(o).__name__}={o.value}"
        if isinstance(a, C.c_void_p):
            if ct is not None and a.value and a.value not in self.labels:      # a host alpha / beta
                if ct == cs.CUDA_R_32F:
                    return f"*{C.c_float.from_address(a.value).value!r}"
                if ct == cs.CUDA_C_64F:
                    return f"*{complex(*(C.c_double * 2).from_address(a.value))!r}"
                return f"*{C.c_double.from_address(a.value).value!r}"
            return self.label(a)
        if isinstance(a, (C.c_int, C.c_long, C.c_ulong, C.c_uint64, C.c_double, C.c_float)):
            return f"{type(a).__name__}={a.value}"
        if isinstance(a, (int, bytes)):
            return repr(a)
        raise TypeError(f"unexpected argument {a!r}")

    def note(self, text, uses=()):
        self.entries.append((text, text, tuple(uses), None))

    def call(self, lib, name, *args):
        scalars, ct = (), None
        for pattern, pos, ctpos in _SCALARS:
            if re.fullmatch(pattern, name):
                scalars, ct = pos, args[ctpos].value
        text = f"{lib}.{name}({', '.join(self._arg(a, ct if i in scalars else None) for i, a in enumerate(args))})"
        uses = tuple(a.value for a in args if isinstance(a, C.c_void_p) and a.value in self.objects)
        destroyed = uses[0] if ("Destroy" in name or name.endswith("_destroyDescr")) and uses else None
        self.entries.append((text, name, uses, destroyed))
        status = self.fail.get(name, 0)
        if status:
            return status
        if name == "b200spmv_last_csr_kernel":
            return b"flat"
        if name.endswith("_get_stats"):
            for v, a in zip((11, 12, 13), args):
                a._obj.value = v
        elif name == "cusparseSpMatGetSize":
            for v, a in zip((4, 5, 6), args[1:]):
                a._obj.value = v
        elif name.endswith("_zeroPivot"):
            self.pivots += 1
            pos, status = (-1, 0) if self.pivots % 2 else (2, cs.CUSPARSE_STATUS_ZERO_PIVOT)
            if isinstance(args[2], _BYREF):
                args[2]._obj.value = pos
            elif args[2].value in self.labels:
                C.c_int.from_address(args[2].value).value = pos
            return status
        else:
            for a in args:
                if isinstance(a, _BYREF) and isinstance(a._obj, C.c_void_p):
                    self.next_object += 0x10
                    a._obj.value = self.next_object
                    self.objects[self.next_object] = self.labels[self.next_object] = \
                        f"{name}@{hashlib.sha1(text.encode()).hexdigest()[:8]}"
                elif isinstance(a, _BYREF) and "bufferSize" in name:
                    a._obj.value = BUFFER_SIZE
        return 0

    # ---- the comparison ---------------------------------------------------------------------------------------------------
    def ordered(self):
        return [text for text, name, _, _ in self.entries if not _is_descriptor_call(name)]

    def descriptor_calls(self):
        return sorted(text for text, name, _, _ in self.entries if _is_descriptor_call(name))

    def released(self):
        return sorted(self.objects[d] for _, _, _, d in self.entries if d is not None)

    def lifecycle_errors(self, exactly_once):
        errors = []
        for obj, label in self.objects.items():
            destroys = [i for i, e in enumerate(self.entries) if e[3] == obj]
            uses = [i for i, e in enumerate(self.entries) if obj in e[2] and e[3] != obj]
            if len(destroys) > 1 or (exactly_once and len(destroys) != 1):
                errors.append(f"{label} destroyed {len(destroys)} times")
            elif destroys and uses and uses[-1] > destroys[0]:
                errors.append(f"{label} used after its destroy")
        return errors


class _Lib:
    def __init__(self, rec, name):
        self._rec, self._name = rec, name

    def __getattr__(self, fn):
        if fn.startswith("__"):
            raise AttributeError(fn)
        return functools.partial(self._rec.call, self._name, fn)


class _Event:
    def __init__(self, rec, name):
        self.rec, self.name = rec, name

    def record(self, stream=None):
        self.rec.note(f"event:{self.name}")


def _run(case, mp):
    """(recorder, result) of one case under the recorders; result: the return label, or the error and what was released."""
    fn, impl, fail = CASES[case]
    rec = _Recorder(fail)
    libs = {k: _Lib(rec, k) for k in ("real", "shim", "spsv")}
    for k, v in libs.items():
        mp.setattr(_lib, k, lambda v=v: v)
    mp.setattr(torch.cuda, "current_stream", lambda *a, **k: types.SimpleNamespace(cuda_stream=STREAM))
    mp.setattr(torch.cuda, "synchronize", lambda *a, **k: rec.note("sync"))
    for f in _FACTORIES:
        mp.setattr(torch, f, functools.wraps(getattr(torch, f))(lambda *a, _f=getattr(torch, f), **k: rec.alloc(_f(*a, **k))))
    clone = torch.Tensor.clone
    mp.setattr(torch.Tensor, "clone", lambda self, *a, **k: rec.alloc(clone(self, *a, **k)))
    api = cs.Api(impl)
    try:
        result = {"ret": rec.label(fn(api, rec))}
    except (cs.CuSparseError, ValueError) as e:
        result = {"error": f"{type(e).__name__}: {e}"}
    gc.collect()                       # a half-built object releases what it holds in __del__
    if "error" in result and fail:
        result["released"] = rec.released()
    return rec, result


def _record(case):
    with pytest.MonkeyPatch.context() as mp:
        rec, result = _run(case, mp)
    if "released" not in result:
        result.update(ordered=rec.ordered(), descriptors=rec.descriptor_calls())
    return result


# ---- the cases ---------------------------------------------------------------------------------------------------------------
ROW, COL, T = cs.CUSPARSE_ORDER_ROW, cs.CUSPARSE_ORDER_COL, cs.CUSPARSE_OPERATION_TRANSPOSE


def _t(r, name, n, dtype=torch.float32, fill=0):
    return r.t(name, torch.full((n,), fill, dtype=dtype))


def _csr(r, rows=4, nnz=6, dtype=torch.float32, batches=1):
    return dict(off=_t(r, "off", (rows + 1) * batches, torch.int32), col=_t(r, "col", nnz * batches, torch.int32),
                val=_t(r, "val", nnz * batches, dtype, 1))


def _coo(r, nnz=6, dtype=torch.float32, batches=1):
    return dict(row=_t(r, "row", nnz * batches, torch.int32), col=_t(r, "col", nnz * batches, torch.int32),
                val=_t(r, "val", nnz * batches, dtype, 1))


def _dense(r, *sizes, dtype=torch.float32):
    return [_t(r, name, n, dtype) for name, n in zip(("B", "C0", "A"), sizes)]


def _events(r):
    return _Event(r, "start"), _Event(r, "stop")


def _spmm(a, r, arrays=None, rows=4, cols=5, n=3, **kw):
    arrays = arrays or _csr(r, rows)
    B, C0 = _dense(r, 64, 64, dtype=arrays["val"].dtype if arrays["val"].dtype != torch.float16 else torch.float32)
    out = cs.spmm(a, rows, cols, arrays, B, C0, kw.pop("alpha", 2.0), kw.pop("beta", 0.5), n=n, **kw)
    assert out is not C0
    return out


def _spmm_bell(a, r, **kw):
    ci, vals = _t(r, "col_ind", 4, torch.int32), _t(r, "values", 32, torch.float16)
    B, C0 = _dense(r, 48, 48, dtype=torch.float16)
    out = cs.spmm_bell(a, 8, 8, 2, 4, ci, vals, B, C0, 3, **kw)
    assert out is C0
    return out


def _spmm_bsr(a, r, batches=1, **kw):
    arrays = dict(off=_t(r, "off", 3 * batches, torch.int32), col=_t(r, "col", 3 * batches, torch.int32),
                  val=_t(r, "val", 48 * batches, torch.float16))
    B, C0 = _dense(r, 96 * batches, 96 * batches, dtype=torch.float16)
    out = cs.spmm_bsr(a, 8, 8, 6, 4, arrays, B, C0, batches=batches, **kw)
    assert out is C0
    return out


def _sddmm(a, r, m=4, n=5, k=3, **kw):
    arrays = _csr(r, m, batches=kw.get("batches", 1))
    A, B = _t(r, "A", 64), _t(r, "B", 64)
    out = cs.sddmm(a, m, n, k, A, B, arrays, kw.pop("alpha", 2.0), kw.pop("beta", 0.5), **kw)
    assert out is arrays["val"]
    return out


def _sddmm_bsr(a, r, batches=1, **kw):
    arrays = dict(off=_t(r, "off", 3 * batches, torch.int32), col=_t(r, "col", 3 * batches, torch.int32),
                  val=_t(r, "val", 48 * batches, torch.bfloat16))
    A, B = _t(r, "A", 96, torch.bfloat16), _t(r, "B", 96, torch.bfloat16)
    out = cs.sddmm_bsr(a, 8, 8, 6, 4, A, B, arrays, 2.0, 0.5, batches=batches, **kw)
    assert out is arrays["val"]
    return out


def _spmv(a, r, fmt, rows=4, cols=5, dtype=torch.float32, close_twice=True, **kw):
    if fmt == "sell":
        arrays = dict(off=_t(r, "off", 3, torch.int32), col=_t(r, "col", 8, torch.int32), val=_t(r, "val", 8, dtype, 1),
                      nnz=6, slice_size=2)
    else:
        arrays = _csr(r, rows, dtype=dtype) if fmt == "csr" else _coo(r, dtype=dtype)
    op = cs.SpMVOperator(a, fmt, rows, cols, arrays, **kw)
    xt, yt = kw.get("xy_dtype") or dtype, kw.get("y_dtype") or kw.get("xy_dtype") or dtype
    x, y = _t(r, "x", 8, xt), _t(r, "y", 8, yt)
    alpha = (2 + 1j) if dtype == torch.complex128 else 2.0
    assert op(x, y, alpha, 0.5) is y
    op.prebuilt(x, y, 3.0, 0.25)()
    attrs = {k: r.label(getattr(op, k)) for k in ("handle", "mat", "vecX", "vecY", "alg", "op", "ctype", "buffer", "buffer_bytes")}
    op.close()
    if close_twice:
        op.close()
    return attrs


def _spsv_solver(a, r):
    arrays = _csr(r, 4, dtype=torch.float64)
    h = a.cusparseCreate()
    first = cs.SpSVSolver(a, 4, arrays, handle=h, device_alpha=True)
    buf = _t(r, "buf", 64, torch.uint8)
    second = cs.SpSVSolver(a, 4, arrays, handle=h, device_alpha=True, mat=first.mat, op=T, buffer=buf,
                           fill=cs.CUSPARSE_FILL_MODE_UPPER, diag=cs.CUSPARSE_DIAG_TYPE_UNIT)
    x, y, alpha = _t(r, "x", 4, torch.float64), _t(r, "y", 4, torch.float64), _t(r, "alpha", 1, torch.float64)
    assert first(x, y, alpha) is y and second(y, x, alpha) is x
    first.update(_t(r, "new_val", 6, torch.float64), cs.CUSPARSE_SPSV_UPDATE_DIAGONAL)
    attrs = {k: r.label(getattr(second, k)) for k in ("handle", "mat", "vecX", "vecY", "descr", "buffer", "buffer_bytes")}
    second.close()
    first.close()
    first.close()
    a.cusparseDestroy(h)
    return attrs


def _spsm_solver(a, r):
    arrays = _csr(r, 4)
    B, C0 = _dense(r, 12, 12)
    s = cs.SpSMSolver(a, 4, arrays, B, C0, 3, op_b=T, order_b=ROW, order_c=ROW, ldc=4, buffer=None, base=1)
    assert s(2.0) is C0
    s.update(_t(r, "new_val", 6), cs.CUSPARSE_SPSM_UPDATE_DIAGONAL)
    attrs = {k: r.label(getattr(s, k)) for k in ("handle", "mat", "descr", "buffer", "B", "C")}
    s.close()
    s.close()
    return attrs


def _csr2csc(a, r, vals=True, **kw):
    arrays = _csr(r, 4, dtype=torch.float64)
    return cs.csr2csc(a, 4, 5, arrays["off"], arrays["col"], arrays["val"] if vals else None, base=1, **kw)


def _coosort(a, r, with_p, **kw):
    rows, cols = _t(r, "rows", 6, torch.int32), _t(r, "cols", 6, torch.int32)
    P = _t(r, "P", 6, torch.int32) if with_p else None
    out = cs.coosort(a, 4, 5, rows, cols, P, **kw)
    assert (out is P) if with_p else out is not None
    return out


def _s2d(a, r, fmt, **kw):
    dense = _t(r, "dense", 40)
    if fmt == cs.CUSPARSE_FORMAT_BLOCKED_ELL:
        a_, b_, vals = _t(r, "colind", 4, torch.int32), None, _t(r, "ellv", 16)
        kw.update(bs=2, ell_cols=4)
    else:
        a_, b_, vals = _t(r, "a", 6, torch.int32), _t(r, "b", 6, torch.int32), _t(r, "vals", 6)
    out = cs.sparse_to_dense(a, fmt, 4, 5, a_, b_, vals, dense, 5, **kw)
    assert out is dense
    return out


def _d2s(a, r, fmt, then=False, **kw):
    dense = _t(r, "dense", 40, torch.float64)
    if then:
        kw["then"] = lambda h, m: r.note(f"then({r.label(h)}, {r.label(m)})", (h.value, m.value))
    if fmt == cs.CUSPARSE_FORMAT_BLOCKED_ELL:
        kw.update(colind=_t(r, "colind", 4, torch.int32), ell_value=_t(r, "ellv", 16, torch.float64), bs=2)
    out = cs.dense_to_sparse(a, fmt, 4, 4, dense, 5, **kw)
    if fmt == cs.CUSPARSE_FORMAT_BLOCKED_ELL:
        assert out is kw["ell_value"]
    return out


def _banded(a, r, penta, buffer="auto"):
    diags = [r.t(f"d{i}", torch.zeros(4, 3, dtype=torch.float64)) for i in range(5 if penta else 3)]
    x = r.t("x", torch.zeros(4, 3, dtype=torch.float64))
    if buffer is True:
        buffer = _t(r, "buf", 64, torch.uint8)
    out = cs.gpsv_interleaved(a, *diags, x, buffer=buffer) if penta else cs.gtsv_interleaved(a, *diags, x, 1, buffer=buffer)
    assert out is x
    return out


def _factor(a, r, fn, **kw):
    arrays = _csr(r, 4, dtype=kw.pop("dtype", torch.float64))
    if isinstance(kw.get("buffer"), bool):
        kw["buffer"] = _t(r, "buf", 64, torch.uint8)
    out = fn(a, 4, arrays["off"], arrays["col"], arrays["val"], **kw)
    assert set(out) <= {"structural", "numerical", "buffer_size"}
    return out


def _stats(a, r):
    out = {}
    for name in ("stats", "spsv_stats", "spsm_stats", "last_csr_kernel"):
        out[name] = getattr(a, name)()
    for name in ("reset_stats", "reset_spsv_stats", "reset_spsm_stats"):
        getattr(a, name)()
    try:
        a.set_option("B200SPMV_CSR_KERNEL", "tile")
        out["set_option"] = "ok"
    except ValueError as e:
        out["set_option"] = str(e)
    return out


def _spmv_batched_csr(a, r, **kw):
    arrays = _csr(r, 4, batches=2)
    B, C0 = _dense(r, 30, 24)
    out = cs.spmm_batched(a, 4, 5, 6, 2, arrays["off"], arrays["col"], arrays["val"], B, C0, 2.0, 0.5, **kw)
    assert out is not C0
    return out


def _spmm_coo_batched(a, r, **kw):
    arrays = _coo(r, batches=2)
    B, C0 = _dense(r, 30, 24)
    out = cs.spmm_coo_batched(a, 4, 5, 6, 2, arrays["row"], arrays["col"], arrays["val"], B, C0, 2.0, 0.5, **kw)
    assert out is not C0
    return out


def _tensor_scalars(r, dtype=torch.float32):
    return dict(alpha=_t(r, "alpha", 1, dtype), beta=_t(r, "beta", 1, dtype))


F = cs.CUSPARSE_FORMAT_CSR, cs.CUSPARSE_FORMAT_CSC, cs.CUSPARSE_FORMAT_COO, cs.CUSPARSE_FORMAT_BLOCKED_ELL
CASES = {
    # name: (case(api, recorder), impl, {function: failing status})
    "spmm_csr": (lambda a, r: _spmm(a, r), "b200", None),
    "spmm_csr_closed": (lambda a, r: _spmm(a, r), "cusparse", None),
    "spmm_coo": (lambda a, r: _spmm(a, r, _coo(r)), "b200", None),
    "spmm_coo_batched_shared": (lambda a, r: _spmm(a, r, dict(_coo(r), nnz=6), batches=2, a_stride=0, b_stride=0), "b200", None),
    "spmm_coo_batched_default": (lambda a, r: _spmm(a, r, _coo(r, batches=2), batches=2), "b200", None),
    "spmm_op_a_t": (lambda a, r: _spmm(a, r, op_a=T, order_b=ROW), "b200", None),
    "spmm_op_b_t": (lambda a, r: _spmm(a, r, op_b=T, order_b=ROW, order_c=ROW), "b200", None),
    "spmm_op_b_t_col": (lambda a, r: _spmm(a, r, op_b=T), "b200", None),
    "spmm_row_ld": (lambda a, r: _spmm(a, r, order_b=ROW, order_c=ROW, ldb=5, ldc=6), "b200", None),
    "spmm_col_ld": (lambda a, r: _spmm(a, r, ldb=7, ldc=8, base=1, alg=cs.CUSPARSE_SPMM_CSR_ALG2), "b200", None),
    "spmm_tensor_alpha": (lambda a, r: _spmm(a, r, **_tensor_scalars(r)), "b200", None),
    "spmm_buffer_none": (lambda a, r: _spmm(a, r, buffer=None), "b200", None),
    "spmm_buffer_given": (lambda a, r: _spmm(a, r, buffer=_t(r, "buf", 64, torch.uint8)), "b200", None),
    "spmm_no_preprocess": (lambda a, r: _spmm(a, r, op_a=T, preprocess=False), "b200", None),
    "spmm_compute_fp64": (lambda a, r: _spmm(a, r, compute=cs.CUDA_R_64F), "b200", None),
    "spmm_half": (lambda a, r: _spmm(a, r, _csr(r, 4, dtype=torch.float16)), "b200", None),
    "spmm_double": (lambda a, r: _spmm(a, r, _csr(r, 4, dtype=torch.float64)), "b200", None),
    "spmm_timing": (lambda a, r: _spmm(a, r, timing=_events(r)), "b200", None),
    "spmm_n_from_b": (lambda a, r: _spmm(a, r, n=None), "b200", None),
    "spmm_coo_batched": (lambda a, r: _spmm_coo_batched(a, r), "b200", None),
    "spmm_coo_batched_broadcast": (lambda a, r: _spmm_coo_batched(a, r, a_stride=0, b_stride=0, order=ROW,
                                                                  alg=cs.CUSPARSE_SPMM_COO_ALG1), "b200", None),
    "spmm_batched": (lambda a, r: _spmv_batched_csr(a, r), "b200", None),
    "spmm_batched_broadcast": (lambda a, r: _spmv_batched_csr(a, r, off_stride=5, colval_stride=0, b_stride=0, order=ROW), "b200", None),
    "spmm_batched_tensor_alpha": (lambda a, r: cs.spmm_batched(a, 4, 5, 6, 1, *_csr(r).values(), *_dense(r, 15, 12),
                                                               **_tensor_scalars(r)), "b200", None),
    "spmm_bell": (lambda a, r: _spmm_bell(a, r), "b200", None),
    "spmm_bell_options": (lambda a, r: _spmm_bell(a, r, order_b=ROW, order_c=ROW, ldb=5, ldc=4, base=1, opB=T, timing=_events(r),
                                                  alg=cs.CUSPARSE_SPMM_BLOCKED_ELL_ALG1, **_tensor_scalars(r)), "b200", None),
    "spmm_bsr": (lambda a, r: _spmm_bsr(a, r, timing=_events(r)), "b200", None),
    "spmm_bsr_batched": (lambda a, r: _spmm_bsr(a, r, batches=2, buffer=None, opB=T, order_c=COL, **_tensor_scalars(r)), "b200", None),
    "spmm_bsr_batched_strides": (lambda a, r: _spmm_bsr(a, r, batches=2, off_stride=3, col_stride=0, val_stride=0, b_stride=0,
                                                        c_stride=50, order_b=COL, ldb=9, ldc=7, compute=cs.CUDA_R_64F,
                                                        alg=cs.CUSPARSE_SPMM_BSR_ALG1, base=1, order_a=COL), "b200", None),
    "sddmm": (lambda a, r: _sddmm(a, r), "b200", None),
    "sddmm_batched_shared": (lambda a, r: _sddmm(a, r, batches=2, a_stride=0, b_stride=0, opA=T, buffer=None, colval_stride=6,
                                                 off_stride=5), "b200", None),
    "sddmm_batched_default": (lambda a, r: _sddmm(a, r, batches=2, order_a=COL, order_b=COL, opB=T), "b200", None),
    "sddmm_options": (lambda a, r: _sddmm(a, r, lda=7, ldb=8, base=1, timing=_events(r), buffer=_t(r, "buf", 64, torch.uint8),
                                          **_tensor_scalars(r)), "b200", None),
    "sddmm_batched": (lambda a, r: cs.sddmm_batched(a, 2, 4, 5, 3, _t(r, "A", 64), _t(r, "B", 64), _csr(r, 4, batches=2),
                                                    alpha=2.0), "b200", None),
    "sddmm_bsr": (lambda a, r: _sddmm_bsr(a, r, timing=_events(r)), "b200", None),
    "sddmm_bsr_batched": (lambda a, r: _sddmm_bsr(a, r, batches=2, a_stride=0, opA=T, order_b=COL, order_c=COL), "b200", None),
    "sddmm_bsr_batched_strides": (lambda a, r: _sddmm_bsr(a, r, batches=2, off_stride=3, col_stride=0, val_stride=48, b_stride=0,
                                                          lda=9, ldb=8, compute=cs.CUDA_R_64F, base=1), "b200", None),
    "spmv_csr": (lambda a, r: _spmv(a, r, "csr"), "b200", None),
    "spmv_csr_closed": (lambda a, r: _spmv(a, r, "csr"), "cusparse", None),
    "spmv_coo_t": (lambda a, r: _spmv(a, r, "coo", op=T, base=1, alg=cs.CUSPARSE_SPMV_COO_ALG2), "b200", None),
    "spmv_sell": (lambda a, r: _spmv(a, r, "sell", alg=cs.CUSPARSE_SPMV_SELL_ALG1), "b200", None),
    "spmv_mixed": (lambda a, r: _spmv(a, r, "csr", xy_dtype=torch.float64, preprocess=False), "b200", None),
    "spmv_half": (lambda a, r: _spmv(a, r, "csr", dtype=torch.float16, y_dtype=torch.float32, compute_dtype=torch.float32),
                  "b200", None),
    "spmv_complex": (lambda a, r: _spmv(a, r, "csr", dtype=torch.complex128, op=cs.CUSPARSE_OPERATION_CONJUGATE_TRANSPOSE),
                     "b200", None),
    "spmv_shared_handle": (lambda a, r: (lambda h: (_spmv(a, r, "csr", handle=h), a.cusparseDestroy(h))[0])(a.cusparseCreate()),
                           "b200", None),
    "spsv_solver": (_spsv_solver, "b200", None),
    "spsv_solver_closed": (_spsv_solver, "cusparse", None),
    "spsv": (lambda a, r: cs.spsv(a, 4, _csr(r, 4), _t(r, "x", 4), 2.0, op=T, base=1), "b200", None),
    "spsm_solver": (_spsm_solver, "b200", None),
    "spsm": (lambda a, r: cs.spsm(a, 4, _csr(r, 4, dtype=torch.float64), _t(r, "B", 12, torch.float64), 3, 2.0), "b200", None),
    "spsm_options": (lambda a, r: cs.spsm(a, 4, _csr(r, 4), _t(r, "B", 24), 3, 2.0, order_c=ROW, ldc=5, order_b=ROW, ldb=6,
                                          device_alpha=True, buffer=_t(r, "buf", 64, torch.uint8)), "b200", None),
    "csr2csc": (lambda a, r: _csr2csc(a, r), "b200", None),
    "csr2csc_symbolic_null": (lambda a, r: _csr2csc(a, r, vals=False, buffer=None), "b200", None),
    "csr2csc_buffer": (lambda a, r: _csr2csc(a, r, buffer=_t(r, "buf", 64, torch.uint8), alg=2), "b200", None),
    "coosort_identity": (lambda a, r: _coosort(a, r, False), "b200", None),
    "coosort_column": (lambda a, r: _coosort(a, r, True, by_row=False, buffer=None), "b200", None),
    "coosort_buffer": (lambda a, r: _coosort(a, r, True, buffer=_t(r, "buf", 64, torch.uint8)), "b200", None),
    "coo2csr": (lambda a, r: cs.coo2csr(a, _t(r, "rows", 6, torch.int32), 4, 1), "b200", None),
    "csr2coo": (lambda a, r: cs.csr2coo(a, _t(r, "off", 5, torch.int32), 6, 1), "b200", None),
    "s2d_csr": (lambda a, r: _s2d(a, r, F[0]), "b200", None),
    "s2d_csc": (lambda a, r: _s2d(a, r, F[1], order=COL, base=1), "b200", None),
    "s2d_coo": (lambda a, r: _s2d(a, r, F[2], nnz=5), "b200", None),
    "s2d_bell": (lambda a, r: _s2d(a, r, F[3], query=False), "b200", None),
    "s2d_csr_no_query": (lambda a, r: _s2d(a, r, F[0], query=False), "b200", None),
    "s2d_bell_query": (lambda a, r: _s2d(a, r, F[3]), "b200", None),
    "d2s_csr": (lambda a, r: _d2s(a, r, F[0]), "b200", None),
    "d2s_csr_then": (lambda a, r: _d2s(a, r, F[0], then=True, order=COL, base=1), "b200", None),
    "d2s_csc_then": (lambda a, r: _d2s(a, r, F[1], then=True), "b200", None),
    "d2s_bell_then": (lambda a, r: _d2s(a, r, F[3], then=True), "b200", None),
    "gpsv": (lambda a, r: _banded(a, r, True), "b200", None),
    "gpsv_buffer": (lambda a, r: _banded(a, r, True, buffer=True), "b200", None),
    "gtsv": (lambda a, r: _banded(a, r, False), "b200", None),
    "gtsv_buffer_none": (lambda a, r: _banded(a, r, False, buffer=None), "b200", None),
    "ilu0_host": (lambda a, r: _factor(a, r, cs.csrilu02), "b200", None),
    "ilu0_host_boost": (lambda a, r: _factor(a, r, cs.csrilu02, boost=(1e-3, 0.5), dtype=torch.float32, base=1,
                                             policy=cs.CUSPARSE_SOLVE_POLICY_NO_LEVEL), "b200", None),
    "ilu0_device_boost_ext": (lambda a, r: _factor(a, r, cs.csrilu02, boost=(1e-3, 0.5), size_call="ext",
                                                   pointer_mode=cs.CUSPARSE_POINTER_MODE_DEVICE), "b200", None),
    "ilu0_buffer": (lambda a, r: _factor(a, r, cs.csrilu02, buffer=True, mat_type=cs.CUSPARSE_MATRIX_TYPE_SYMMETRIC), "b200", None),
    "ilu0_buffer_none": (lambda a, r: _factor(a, r, cs.csrilu02, buffer=None), "b200", None),
    "ic0": (lambda a, r: _factor(a, r, cs.csric02, dtype=torch.float32), "b200", None),
    "ic0_device_ext": (lambda a, r: _factor(a, r, cs.csric02, size_call="ext", pointer_mode=cs.CUSPARSE_POINTER_MODE_DEVICE),
                       "b200", None),
    "stats": (_stats, "b200", None),
    "stats_closed": (_stats, "cusparse", None),
    "fail_spmm": (lambda a, r: _spmm(a, r, _coo(r)), "b200", {"cusparseSpMM": 7}),
    "fail_spmm_batched": (lambda a, r: _spmv_batched_csr(a, r), "b200", {"cusparseSpMM": 7}),
    "fail_sddmm": (lambda a, r: _sddmm(a, r), "b200", {"cusparseSDDMM": 8}),
    "fail_spmm_bsr": (lambda a, r: _spmm_bsr(a, r), "b200", {"cusparseSpMM": 3}),
    "fail_csr2csc": (lambda a, r: _csr2csc(a, r), "b200", {"cusparseCsr2cscEx2": 11}),
    "fail_s2d": (lambda a, r: _s2d(a, r, F[0]), "b200", {"cusparseSparseToDense": 10}),
    "fail_spsv_analysis": (lambda a, r: cs.spsv(a, 4, _csr(r, 4), _t(r, "x", 4)), "b200", {"cusparseSpSV_analysis": 6}),
    "fail_spsv_solver_analysis": (lambda a, r: cs.SpSVSolver(a, 4, _csr(r, 4), device_alpha=True), "b200",
                                  {"cusparseSpSV_analysis": 6}),
}


@pytest.fixture(scope="module")
def golden():
    with open(GOLDEN) as f:
        return json.load(f)


def test_golden_covers_every_case(golden):
    assert sorted(golden) == sorted(CASES)


@pytest.mark.parametrize("case", sorted(CASES))
def test_trace_matches_golden(case, golden, monkeypatch):
    rec, result = _run(case, monkeypatch)
    want = golden[case]
    if CASES[case][2]:                                  # a failing call
        assert result["error"] == want["error"]
        assert rec.lifecycle_errors(exactly_once=False) == []
        missing = collections.Counter(want["released"]) - collections.Counter(result["released"])
        assert not missing, f"released less than before: {sorted(missing.elements())}"
        return
    assert result == {k: want[k] for k in result}
    ordered = rec.ordered()
    if case in DEVICE_MODE_ADDED and ordered != want["ordered"]:
        assert re.fullmatch(r"real\.cusparseSetPointerMode\(cusparseCreate@\w+, c_int=1\)", ordered.pop(2))
    assert ordered == want["ordered"]
    assert rec.descriptor_calls() == want["descriptors"]
    assert rec.lifecycle_errors(exactly_once=True) == []


if __name__ == "__main__":
    if len(sys.argv) != 3 or sys.argv[1] != "--record":
        sys.exit(f"usage: {sys.argv[0]} --record PATH")
    with open(sys.argv[2], "w") as f:
        json.dump({case: _record(case) for case in sorted(CASES)}, f, indent=1, sort_keys=True)
        f.write("\n")
