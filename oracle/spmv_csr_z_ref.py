"""oracle/spmv_csr_z_ref.py -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

Fixtures for the double-complex CSR SpMV y = alpha * op(A) * x + beta * y (spmv_csr_z.cu): A rows x cols CSR (`off`, `col` with index
base `base`, complex values), x, y, alpha, beta complex, CUDA_C_64F compute, op "N", "T" or "C".

* `reference_int`: the exact result for Gaussian-integer data, in Python ints.  Its precondition check asserts that every partial
  result the kernel can form stays below 2^53 in magnitude, so every fp64 product, fma and sum on the device is exact and any correct
  kernel returns the reference bit for bit, whatever its summation order (N, T and C alike).
* `fma`: a correctly rounded fused multiply-add, float(Fraction(a) * Fraction(b) + Fraction(c)), with IEEE-754's signs of zero.
* `restate_n`: the kernel's opA = N arithmetic restated in fp64 for any data: the fixed complex product, run sums, piece sums, the
  pieces in ascending chunk order and the fixed epilogue.  It gives the kernel's bits.
* `walk`: both walks' work split, shared with the half-precision kernel (oracle/spmv_csr16_ref.py): the same chunking, pieces and carry
  slots.
"""
from __future__ import annotations

import ctypes as C
import math
from fractions import Fraction

import numpy as np

from oracle.spmm_csr16_ref import pattern  # noqa: F401  (the same CSR pattern helper)
from oracle.spmv_csr16_ref import slot, walk  # noqa: F401  (the same work split)

EXACT = 1 << 53


def params(lib=None) -> dict:
    if lib is None:
        from cudalibrarysamples_b200 import lib as _lib
        lib = _lib.shim()
    v = [C.c_int32() for _ in range(3)]
    lib.b200spmv_csr_z_params(*[C.byref(x) for x in v])
    return dict(zip(("chunk", "run", "warps"), (x.value for x in v)))


def values(rows, cols, nnz, seed, lo=-2, hi=2):
    """Gaussian-integer (complex128 with integer parts) values of A (nnz), x (cols) and y0 (rows) in [lo, hi] + i [lo, hi]"""
    rng = np.random.default_rng(seed)

    def z(n):
        return rng.integers(lo, hi + 1, n).astype(np.float64) + 1j * rng.integers(lo, hi + 1, n).astype(np.float64)
    return z(nnz), z(cols), z(rows)


# ------------------------------------------------------------------------------------------------ exact reference
def _gi(v) -> tuple[int, int]:
    v = complex(v)
    assert v.real == int(v.real) and v.imag == int(v.imag), v
    return int(v.real), int(v.imag)


def _mul(a, b):
    return a[0] * b[0] - a[1] * b[1], a[0] * b[1] + a[1] * b[0]


def _mag(a):
    return abs(a[0]) + abs(a[1])


def reference_int(off, col, val, x, y0, alpha, beta, op="N", base=0, cols=None) -> np.ndarray:
    """alpha * op(A) @ x + beta * y0 as complex128 (exact), after checking that every value the kernel forms is an integer below 2^53;
    beta == 0 ignores y0 (it may be None or hold NaN).  y has rows entries for op "N", `cols` entries for "T" / "C"."""
    off = [int(o) - base for o in off]
    col = [int(c) - base for c in col]
    rows = len(off) - 1
    ny = rows if op == "N" else cols
    al, be = _gi(alpha), _gi(beta)
    acc = [(0, 0)] * ny
    bound = [0] * ny                                  # sum of |re| + |im| of every term: bounds each partial sum in any order
    for r in range(rows):
        for k in range(off[r], off[r + 1]):
            v = _gi(val[k])
            if op == "C":
                v = (v[0], -v[1])
            if op == "N":
                p = _mul(v, _gi(x[col[k]]))
                i = r
            else:                                     # the scatter adds alpha * (v * x[r]) into y[c]
                vx = _mul(v, _gi(x[r]))
                assert _mag(vx) < EXACT
                p = _mul(al, vx)
                i = col[k]
            acc[i] = (acc[i][0] + p[0], acc[i][1] + p[1])
            bound[i] += _mag(p)
    out = np.zeros(ny, np.complex128)
    for i in range(ny):
        a = _mul(al, acc[i]) if op == "N" else acc[i]
        t = (0, 0) if be == (0, 0) else _mul(be, _gi(y0[i]))
        big = (_mag(al) * bound[i] if op == "N" else bound[i]) + _mag(t)
        assert bound[i] < EXACT and big < EXACT, "a product, partial sum or epilogue term would leave fp64's exact integers"
        out[i] = complex(a[0] + t[0], a[1] + t[1])
    return out


# ------------------------------------------------------------------------------------------------ the kernel's arithmetic
def fma(a: float, b: float, c: float) -> float:
    """a * b + c rounded once to fp64 (round to nearest even), with IEEE-754's sign of an exact zero"""
    if not (math.isfinite(a) and math.isfinite(b) and math.isfinite(c)):
        return a * b + c                              # inf / NaN: the unfused form gives the same result
    exact = Fraction(a) * Fraction(b) + Fraction(c)
    if exact != 0:
        return float(exact)
    p_neg = (math.copysign(1.0, a) < 0) != (math.copysign(1.0, b) < 0)
    p_zero = a == 0 or b == 0
    if p_zero and c == 0:                             # (+-0) + (+-0): -0 only when both are -0
        return -0.0 if p_neg and math.copysign(1.0, c) < 0 else 0.0
    return 0.0                                        # an exact cancellation rounds to +0


def cmul(a: complex, b: complex) -> complex:
    """the kernel's product: (fma(ar, br, -(ai * bi)), fma(ar, bi, ai * br))"""
    return complex(fma(a.real, b.real, -(a.imag * b.imag)), fma(a.real, b.imag, a.imag * b.real))


def cadd(a: complex, b: complex) -> complex:
    return complex(a.real + b.real, a.imag + b.imag)


def epilogue(acc: complex, alpha: complex, beta: complex, y: complex | None) -> complex:
    """(fma(al_r, acc_r, fma(-al_i, acc_i, t_r)), fma(al_r, acc_i, fma(al_i, acc_r, t_i))), t = beta * y; beta == 0: t = 0, y unread"""
    t = 0j if beta == 0 else cmul(beta, y)
    return complex(fma(alpha.real, acc.real, fma(-alpha.imag, acc.imag, t.real)),
                   fma(alpha.real, acc.imag, fma(alpha.imag, acc.real, t.imag)))


def piece(prods, s, e, run) -> complex:
    """S of the piece [s, e) of one row inside one chunk (entry indices): 0 + each run segment's sum in ascending order, a segment
    summed as 0 + its products in order (a whole run's sum is the run sum the kernel reads back)"""
    acc = 0j
    p = s
    while p < e:
        q = min(e, (p // run + 1) * run)
        u = 0j
        for i in range(p, q):
            u = cadd(u, prods[i])
        acc = cadd(acc, u)
        p = q
    return acc


def restate_n(off, col, val, x, y0, alpha, beta, chunk, run, base=0) -> np.ndarray:
    """y as b200spmv_csr_z computes it for op = N (either walk), in fp64: every row's pieces in ascending chunk order, acc = 0 + S0 +
    S1 + ..., then the epilogue; Python floats are IEEE doubles, so this is bit for bit"""
    off = [int(o) - base for o in off]
    col = [int(c) - base for c in col]
    rows = len(off) - 1
    alpha, beta = complex(alpha), complex(beta)
    prods = [cmul(complex(val[k]), complex(x[col[k]])) for k in range(len(col))]
    out = np.zeros(rows, np.complex128)
    for r in range(rows):
        rs, re = off[r], off[r + 1]
        acc = 0j
        c = rs // chunk
        while c * chunk < re:
            acc = cadd(acc, piece(prods, max(rs, c * chunk), min(re, (c + 1) * chunk), run))
            c += 1
        out[r] = epilogue(acc, alpha, beta, None if beta == 0 else complex(y0[r]))
    return out
