"""numpy restatement of the batched banded solves (batched_banded.cu, DESIGN.md 3.25), one system at a time.

Arrays are interleaved as cusparse<t>gpsvInterleavedBatch / gtsvInterleavedBatch take them: shape (m, batch), element i of system j
at [i, j].  The diagonals are given sub-diagonals first -- (ds, dl, d, du, dw) for the pentadiagonal solve, (dl, d, du) for the
tridiagonal one -- and slot i of a diagonal is the coefficient in row i.  The steps are the kernels': Givens QR with a real c and a
complex s (gpsv, gtsv algo 2), LU with partial pivoting (gtsv algo 1), Thomas without pivoting (gtsv algo 0); the out-of-band slots
are never read.  tests/test_banded_cpu.py checks these against scipy.linalg.solve_banded and the kernels' own source against them.
"""
from __future__ import annotations

import json
import os

import numpy as np

GOLDEN = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "gpsv_sample.json")
GIVENS, PIVOT_LU, THOMAS = "givens", "pivot_lu", "thomas"
GTSV_METHOD = {0: THOMAS, 1: PIVOT_LU, 2: GIVENS}


def sample() -> dict:
    """cuSPARSE/gpsvInterleavedBatch's two 4 x 4 systems (ds, dl, d, du, dw, b as the sample aggregates them: system after
    system) and their solution, computed in float64."""
    with open(GOLDEN) as f:
        return json.load(f)


def band_mask(m: int, P: int) -> np.ndarray:
    """(2P + 1, m): True where slot i of diagonal o is inside the matrix (row i, column i - P + o)"""
    i = np.arange(m)[None, :]
    c = i - P + np.arange(2 * P + 1)[:, None]
    return (c >= 0) & (c < m)


def dense(diags, j: int = 0) -> np.ndarray:
    """System j of the interleaved diagonals as a dense m x m matrix (out-of-band slots ignored)."""
    P = (len(diags) - 1) // 2
    m = diags[0].shape[0]
    A = np.zeros((m, m), dtype=np.result_type(*[d.dtype for d in diags], np.float64))
    mask = band_mask(m, P)
    for o, d in enumerate(diags):
        for i in range(m):
            if mask[o, i]:
                A[i, i - P + o] = d[i, j]
    return A


def banded_ab(diags, j: int = 0) -> np.ndarray:
    """System j in scipy.linalg.solve_banded's (P, P) storage: ab[P + i - c, c] = A[i, c]."""
    P = (len(diags) - 1) // 2
    m = diags[0].shape[0]
    ab = np.zeros((2 * P + 1, m), dtype=np.result_type(*[d.dtype for d in diags], np.float64))
    mask = band_mask(m, P)
    for o, d in enumerate(diags):
        for i in range(m):
            if mask[o, i]:
                ab[2 * P - o, i - P + o] = d[i, j]
    return ab


def _abs1(v):
    return abs(v.real) + abs(v.imag)


def _rdiv(v, d):
    """v / d for a real d, part by part (numpy's complex division forms 1 / d, which overflows for a subnormal d)"""
    if not np.iscomplexobj(v):
        return v / d
    return type(v)(v.real / d + 1j * (v.imag / d))


def _div(a, b):
    """a / b, for complex values by Smith's method as the kernels compute it"""
    if not np.iscomplexobj(a):
        return a / b
    if abs(b.real) >= abs(b.imag):
        r = b.imag / b.real
        d = b.real + b.imag * r
        return type(a)((a.real + a.imag * r) / d + 1j * ((a.imag - a.real * r) / d))
    r = b.real / b.imag
    d = b.real * r + b.imag
    return type(a)((a.real * r + a.imag) / d + 1j * ((a.imag * r - a.real) / d))


def solve_system(diags, b, method: str, dtype=None):
    """One system: diags a list of 2P + 1 length-m vectors, b length m.  Returns x in `dtype` arithmetic (default: b's)."""
    dtype = np.dtype(dtype or b.dtype)
    rdt = np.zeros(1, dtype).real.dtype.type
    P = (len(diags) - 1) // 2
    m = b.shape[0]
    W = P if method == THOMAS else 2 * P
    mask = band_mask(m, P)
    zero = dtype.type(0)

    def row(i):
        if i >= m:
            return [zero] * (2 * P + 1), zero
        return [dtype.type(diags[o][i]) if mask[o, i] else zero for o in range(2 * P + 1)], dtype.type(b[i])

    r = [[zero] * (2 * P + 1) for _ in range(P + 1)]
    rb = [zero] * (P + 1)

    def shift_in(i):
        for q in range(P):
            r[q] = r[q + 1][1:] + [zero]
            rb[q] = rb[q + 1]
        r[P], rb[P] = row(i)

    for i in range(P + 1):
        shift_in(i)
    U = np.zeros((m, W), dtype)
    y = np.zeros(m, dtype)
    for k in range(m):
        for q in range(1, P + 1):
            top, bot = r[0][0], r[q][0]
            if bot == 0:
                continue
            if method == GIVENS:
                at = rdt(abs(top))
                n = rdt(np.hypot(at, rdt(abs(bot))))
                c = at / n
                ph = dtype.type(1) if at == 0 else (_rdiv(top, at) if np.iscomplexobj(top) else dtype.type(1 if top > 0 else -1))
                s = ph * _rdiv(np.conj(bot), n)
                ms = -np.conj(s)
                r[0], r[q] = [c * p + s * t for p, t in zip(r[0], r[q])], [ms * p + c * t for p, t in zip(r[0], r[q])]
                r[q][0] = zero
                rb[0], rb[q] = c * rb[0] + s * rb[q], ms * rb[0] + c * rb[q]
            else:
                if method == PIVOT_LU and _abs1(bot) > _abs1(top):
                    r[0], r[q] = r[q], r[0]
                    rb[0], rb[q] = rb[q], rb[0]
                lq = _div(r[q][0], r[0][0])
                r[q] = [zero] + [t - lq * p for p, t in zip(r[0][1:], r[q][1:])]
                rb[q] = rb[q] - lq * rb[0]
        U[k] = [_div(r[0][q], r[0][0]) for q in range(1, W + 1)]
        y[k] = _div(rb[0], r[0][0])
        shift_in(k + 1 + P)
    x = np.zeros(m, dtype)
    for k in range(m - 1, -1, -1):
        v = y[k]
        for q in range(1, W + 1):
            if k + q < m:
                v = v - U[k, q - 1] * x[k + q]
        x[k] = v
    return x


def solve(diags, x, method: str, dtype=None) -> np.ndarray:
    """Every system of the interleaved (m, batch) arrays; returns the (m, batch) solutions."""
    return np.stack([solve_system([d[:, j] for d in diags], x[:, j], method, dtype) for j in range(x.shape[1])], axis=1)


def backward_error(diags, x, b) -> np.ndarray:
    """Per system: ||b - A x||_inf / (||A||_inf ||x||_inf), in float64 / complex128."""
    out = []
    for j in range(x.shape[1]):
        A = dense([d.astype(np.complex128) for d in diags], j)
        xj = x[:, j].astype(np.complex128)
        r = b[:, j].astype(np.complex128) - A @ xj
        out.append(np.abs(r).max() / max(np.abs(A).sum(1).max() * np.abs(xj).max(), np.finfo(float).tiny))
    return np.array(out)


if __name__ == "__main__":
    # writes tests/golden/gpsv_sample.json from the arrays of cuSPARSE/gpsvInterleavedBatch/gpsvInterleavedBatch_example.c
    import scipy.linalg
    n, batch = 4, 2
    S = [0, 0, 11, 12, 0, 0, 25, 26]
    L = [0, 5, 6, 7, 0, 19, 20, 21]
    M = [1, 2, 3, 4, 15, 16, 17, 18]
    U = [8, 9, 10, 0, 22, 23, 24, 0]
    Wd = [13, 14, 0, 0, 27, 28, 0, 0]
    B = [1, 2, 3, 4, 5, 6, 7, 8]
    inter = lambda v: np.array(v, float).reshape(batch, n).T          # noqa: E731
    diags = [inter(v) for v in (S, L, M, U, Wd)]
    X = np.stack([scipy.linalg.solve_banded((2, 2), banded_ab(diags, j), inter(B)[:, j]) for j in range(batch)], axis=1)
    json.dump(dict(source="cuSPARSE/gpsvInterleavedBatch/gpsvInterleavedBatch_example.c", m=n, batch=batch,
                   layout="aggregate: system after system, as the sample's host arrays", ds=S, dl=L, d=M, du=U, dw=Wd, b=B,
                   x=X.T.reshape(-1).tolist(),
                   x_printed=[-0.0592, 0.3428, -0.1295, 0.1982, -0.0012, 0.2792, -0.0416, 0.0898]),
              open(GOLDEN, "w"), indent=1)
    print("wrote", GOLDEN)
