"""oracle/bicgstab_ref.py -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

Unpreconditioned BiCGStab in numpy float64, two ways:

  * `sample_loop`: a literal transcription of the loop of cuSPARSE/bicgstab/bicgstab_example.c:212-351 with M = I (the two
    triangular solves become copies), step by step in the sample's order: the dots, the axpy / scal sequence, the host-side
    scalars and the two `nrm < threshold` exits.  No breakdown handling, as in the sample.
  * `fused`: the iteration as the kernels of cudalibrarysamples_b200/csrc/bicgstab_fused.cu take it (one scalar per state
    slot, the status protocol included: convergence at s or at r, the breakdowns, the counter and the residual history).

On systems without a breakdown the two agree bit for bit: every vector element sees the same roundings in the same order and
every dot is the same np.dot.  The GPU result differs from `fused` by summation order and fused multiply-adds only.

`kernel_reference` gives the exact result of each kernel on the integer / dyadic fixtures (`KERNELS`, `SCALARS`) that the GPU
tests drive through the C ABI at the sizes of oracle.exact.cg_sizes.
"""
from __future__ import annotations

import math
from fractions import Fraction

import numpy as np

from oracle import exact as E

# the status codes and slot indices of include/b200spmv.h (tests/test_bicgstab_cpu.py checks them against the header)
RUNNING, CONVERGED_S, CONVERGED_R = 0, 1, 2
BREAKDOWN_DENOM, BREAKDOWN_TT, BREAKDOWN_OMEGA, BREAKDOWN_RHO, BREAKDOWN_NONFINITE = 3, 4, 5, 6, 7
STATUS_NAMES = {RUNNING: "running", CONVERGED_S: "converged_s", CONVERGED_R: "converged_r", BREAKDOWN_DENOM: "breakdown_denom",
                BREAKDOWN_TT: "breakdown_tt", BREAKDOWN_OMEGA: "breakdown_omega", BREAKDOWN_RHO: "breakdown_rho",
                BREAKDOWN_NONFINITE: "breakdown_nonfinite"}
SLOTS = dict(RHO=0, ALPHA=1, OMEGA=2, DENOM=3, S2=4, TS=5, TT=6, RHO_NEW=7, R2=8, THRESHOLD=9)


def sample_loop(A, b, max_iters, tol, x0=None):
    """bicgstab_example.c:183-351 with M = I.  Returns dict(x, iterations, history, exit) -- history[k] is the nrm_R the
    sample prints at the start of iteration k + 1 (nrm_S when it leaves at step 13), exit: "s", "r" or None."""
    x = np.zeros_like(b) if x0 is None else x0.copy()
    R0 = b.copy()                                                   # ### 1 ### R0 = b - A X0
    R0 = -1.0 * (A @ x) + 1.0 * R0 if x0 is not None else R0
    delta = np.dot(R0, R0)
    delta_prev = delta
    R = R0.copy()
    nrm_R = np.linalg.norm(R0)
    threshold = tol * nrm_R
    history = [nrm_R]
    P = V = None
    alpha = omega = 0.0
    for i in range(1, max_iters + 1):
        if i == 1:
            P = R.copy()                                            # ### 4, 7 ###
        else:
            delta = np.dot(R0, R)                                   # ### 6 ###
            beta = (delta / delta_prev) * (alpha / omega)
            delta_prev = delta
            P = (-omega) * V + P                                    # ### 7 ### (a) axpy
            P = beta * P                                            #           (b) scal
            P = 1.0 * R + P                                         #           (c) axpy
        P_aux = P.copy()                                            # ### 9 ### M = I
        V = A @ P_aux                                               # ### 10 ###
        denominator = np.dot(R0, V)
        alpha = delta / denominator
        x = alpha * P_aux + x                                       # ### 11 ###
        S = R.copy()                                                # ### 12 ###
        S = (-alpha) * V + S
        nrm_S = np.linalg.norm(S)                                   # ### 13 ###
        if nrm_S < threshold:
            history.append(nrm_S)
            return dict(x=x, iterations=i, history=history, exit="s")
        S_aux = S.copy()                                            # ### 14 ### M = I
        T = A @ S_aux                                               # ### 15 ###
        omega_num = np.dot(T, S)
        omega_den = np.dot(T, T)
        omega = omega_num / omega_den
        x = omega * S_aux + x                                       # ### 16 ###
        R = S.copy()                                                # ### 17 ###
        R = (-omega) * T + R
        nrm_R = np.linalg.norm(R)                                   # ### 18 ###
        history.append(nrm_R)
        if nrm_R < threshold:
            return dict(x=x, iterations=i, history=history, exit="r")
    return dict(x=x, iterations=max_iters, history=history, exit=None)


def _finite(*v):
    return all(math.isfinite(float(a)) for a in v)


def fused(matvec, b, max_iters, tol=None, x0=None, dot=np.dot):
    """The fused solver's iteration (bicgstab_fused.cu), status protocol included.  matvec(v) -> A v; dot(a, b) -> a . b
    (the gloo tests pass an all-reduced dot).  Returns dict(x, status, iterations, history)."""
    x = np.zeros_like(b) if x0 is None else x0.copy()
    r0 = b - matvec(x) if x0 is not None else b.copy()
    rho_new = dot(r0, r0)                                           # b200cg_dot + b200bicgstab_init
    r, p = r0.copy(), r0.copy()
    rho, r2 = rho_new, rho_new
    threshold = -1.0 if tol is None else tol * math.sqrt(rho)
    history = [math.sqrt(rho)]
    status = BREAKDOWN_NONFINITE if not _finite(rho) else CONVERGED_R if rho == 0 else RUNNING
    k = 0

    def out():
        return dict(x=x, status=status, iterations=k, history=history)

    for _ in range(max_iters):
        if status != RUNNING:
            break
        v = matvec(p)
        denom = dot(r0, v)
        alpha = rho_new / denom                                     # update_s
        if denom == 0:
            status = BREAKDOWN_DENOM
            break
        if not _finite(alpha):
            status = BREAKDOWN_NONFINITE
            break
        s = r - alpha * v
        s2 = dot(s, s)
        rho = rho_new
        t = matvec(s)
        ts, tt = dot(t, s), dot(t, t)                               # dot2
        if not _finite(s2):                                         # update_xr
            status = BREAKDOWN_NONFINITE
            break
        if math.sqrt(s2) < threshold:
            x = x + alpha * p
            r = s.copy()
            rho_new, r2 = dot(r0, r), dot(r, r)
            k += 1
            history.append(math.sqrt(s2))
            status = CONVERGED_S
            break
        omega = ts / tt
        if not _finite(ts, tt):
            status = BREAKDOWN_NONFINITE
        elif tt == 0:
            status = BREAKDOWN_TT
        elif not _finite(omega):
            status = BREAKDOWN_NONFINITE
        elif omega == 0:
            status = BREAKDOWN_OMEGA
        if status != RUNNING:
            break
        x = (x + alpha * p) + omega * s
        r = s - omega * t
        rho_new, r2 = dot(r0, r), dot(r, r)
        k += 1                                                      # update_p
        history.append(math.sqrt(r2) if r2 >= 0 else float("nan"))
        beta = (rho_new / rho) * (alpha / omega)
        if not _finite(r2, rho_new):
            status = BREAKDOWN_NONFINITE
        elif math.sqrt(r2) < threshold:
            status = CONVERGED_R
        elif rho_new == 0:
            status = BREAKDOWN_RHO
        elif not _finite(beta):
            status = BREAKDOWN_NONFINITE
        if status != RUNNING:
            break
        p = r + beta * (p - omega * v)
    return out()


# ------------------------------------------------------------------------------------------------ exact kernel fixtures
# Device scalars whose quotients are dyadic: alpha = rho_new / denom = -1/4, omega = ts / tt = 1/2,
# beta = (rho_new / rho) (alpha / omega) = (1/2) (-1/2) = -1/4; threshold -1: no convergence test.
SCALARS = dict(RHO=3.0, ALPHA=-0.25, OMEGA=0.5, DENOM=-12.0, S2=5.0, TS=1.5, TT=3.0, RHO_NEW=3.0, R2=7.0, THRESHOLD=-1.0)
SCALARS_P = dict(SCALARS, RHO_NEW=1.5)                              # update_p: rho_new / rho = 1/2

KERNELS = {  # name: (vector arguments in call order, vectors written, state slots reduced)
    "init": (["r0", "r", "p"], ["r", "p"], []),
    "update_s": (["r", "v", "s"], ["s"], ["S2"]),
    "dot2": (["t", "s"], [], ["TS", "TT"]),
    "update_xr": (["x", "r", "p", "s", "t", "r0"], ["x", "r"], ["RHO_NEW", "R2"]),
    "update_p": (["p", "r", "v"], ["p"], []),
}


def kernel_scalars(name):
    return SCALARS_P if name == "update_p" else SCALARS


def kernel_vectors(kind, n, name, seed):
    """int64 vectors of n nonzero integers for kernel `name` (|v| in the kind's range of oracle.exact)"""
    return E.cg_vectors(kind, n, KERNELS[name][0], seed)


def _q(v):
    return Fraction(v).limit_denominator(1 << 20)


def _vec(num, den):
    assert np.all(np.abs(num) < (1 << 53)), "a result needs more than 53 bits"
    return np.asarray(num, np.int64).astype(np.float64) / den


def _sum(terms, den):
    """sum of int64 terms / den, asserting that every partial sum in any order is exact (sum |terms| < 2^53)"""
    assert int(np.abs(terms).sum()) < (1 << 53)
    return float(int(terms.sum())) / den


def kernel_reference(name, v, scal=None):
    """What kernel `name` must write from the int64 vectors v and the state scalars: {vector or slot: float64}, computed in
    integers (every element is an integer over 2, 4 or 8 and every reduction exact).  init is checked separately (copies)."""
    scal = scal or kernel_scalars(name)
    alpha = _q(scal["RHO_NEW"]) / _q(scal["DENOM"]) if name == "update_s" else _q(scal["ALPHA"])
    omega = _q(scal["TS"]) / _q(scal["TT"]) if name == "update_xr" else _q(scal["OMEGA"])
    out = {}
    if name == "update_s":
        assert alpha == Fraction(-1, 4)
        s4 = 4 * v["r"] + v["v"]                                    # 4 (r - alpha v)
        out["s"] = _vec(s4, 4)
        out["S2"] = _sum(s4 * s4, 16)
    elif name == "dot2":
        out["TS"] = _sum(v["t"] * v["s"], 1)
        out["TT"] = _sum(v["t"] * v["t"], 1)
    elif name == "update_xr":
        assert alpha == Fraction(-1, 4) and omega == Fraction(1, 2)
        out["x"] = _vec(4 * v["x"] - v["p"] + 2 * v["s"], 4)        # x + alpha p + omega s
        r2x = 2 * v["s"] - v["t"]                                   # 2 (s - omega t)
        out["r"] = _vec(r2x, 2)
        out["RHO_NEW"] = _sum(v["r0"] * r2x, 2)
        out["R2"] = _sum(r2x * r2x, 4)
    elif name == "update_p":
        beta = (_q(scal["RHO_NEW"]) / _q(scal["RHO"])) * (alpha / omega)
        assert beta == Fraction(-1, 4) and omega == Fraction(1, 2)
        out["p"] = _vec(8 * v["r"] - 2 * v["p"] + v["v"], 8)      # r + beta (p - omega v)
    elif name == "init":
        out["r"] = v["r0"].astype(np.float64)
        out["p"] = v["r0"].astype(np.float64)
    return out
