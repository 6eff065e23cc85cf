"""oracle/exact.py -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

Exact fixtures for SpMV / SpMM: integer-valued inputs on which every partial sum, in any order, is an integer that the value
type represents exactly.  Any correct kernel then returns the exact result, whatever its summation order, its atomics or its
split of a row between warps, CTAs and tiles -- so the kernels are compared with a plain integer reference BIT FOR BIT instead of
against a tolerance, and a dropped, duplicated or narrowed product always shows.

  * A and x hold NONZERO small integers (+-1 .. +-4): a dropped or duplicated product always changes the row sum;
  * alpha and beta are powers of two (or 0 / +-1), y0 holds even integers: alpha * S + beta * y0 is a multiple of 1/2;
  * the "wide" fp64 variant takes values of 12-13 bits, so products need 24-26 bits and row sums more than fp32 has, while
    staying below 2^53: an accumulator narrowed to fp32 loses bits;
  * the "mixed" variant (fp32 A, fp64 x / y / arithmetic) keeps A small (exact in fp32) and makes x 30-31 bits wide.

The reference is computed in int64 (`reference`), and `check_exact` asserts the exactness precondition row by row:
sum |products| and 2 * (|alpha| * sum |products| + |beta * y0|) stay below 2^p (p = 24 for fp32 arithmetic, 53 for fp64).

The boundary profiles are row-length sequences built from the kernels' own constants (read from the built library by
`kernel_params`), and `coverage` recomputes from the row offsets which boundary class a matrix actually hits.

The fused CG BLAS-1 kernels (cg_fused.cu) get the same treatment at the end of this file: vectors of nonzero integers, device
scalars whose quotients are powers of two (alpha = -1/4, beta = 1/2), an int64 reference on values scaled by 4 (vectors) and
16 (r . r), edge sizes built from `cg_params`, and `cg_walk` / `cg_coverage`, a model of the kernels' index mapping.
"""
from __future__ import annotations

import ctypes as C
from fractions import Fraction

import numpy as np

MANTISSA = {"f32": 24, "f64": 53, "wide": 53, "mixed": 53}
# (alpha, beta); beta == 0 is run on a NaN-filled y
SCALARS = [(1.0, 0.0), (-2.0, 0.5), (-2.0, 1.0), (0.5, -1.0)]


# ------------------------------------------------------------------------------------------------ the kernels' constants
def kernel_params(lib=None) -> dict:
    """The tile / flat / short constants of the built product library (b200spmv_csr_plan_params, _flat_params, _short_params)."""
    if lib is None:
        from cudalibrarysamples_b200 import lib as _lib
        lib = _lib.shim()
    t, l, b = C.c_int32(), C.c_int32(), C.c_int32()
    lib.b200spmv_csr_plan_params(C.byref(t), C.byref(l), C.byref(b))
    wc, cta, pc = C.c_int32(), C.c_int32(), C.c_int32()
    lib.b200spmv_csr_flat_params(C.byref(wc), C.byref(cta), C.byref(pc))
    cap, rpw = C.c_int32(), C.c_int32()
    lib.b200spmv_csr_short_params(C.byref(cap), C.byref(rpw))
    return dict(tile=t.value, long_row=l.value, block=b.value, warp_chunk=wc.value, cta_nnz=cta.value, plan_chunk=pc.value,
                short_cap=cap.value, short_rows=rpw.value)


# ------------------------------------------------------------------------------------------------ values
def nonzero_ints(rng, n, lo, hi):
    """n integers with lo <= |v| < hi and a random sign (lo >= 1: never zero)"""
    return rng.integers(lo, hi, n, dtype=np.int64) * rng.choice(np.array([-1, 1], np.int64), n)


_RANGES = {  # kind -> ((|A| range), (|x| range), (|y0| / 2 range))
    "f32": ((1, 5), (1, 5), (0, 33)),
    "f64": ((1, 5), (1, 5), (0, 33)),
    "wide": ((1 << 12, 1 << 13), (1 << 12, 1 << 13), (0, 1 << 30)),
    "mixed": ((1, 5), (1 << 30, 1 << 31), (0, 1 << 30)),
}
NP_A = {"f32": np.float32, "f64": np.float64, "wide": np.float64, "mixed": np.float32}
NP_XY = {"f32": np.float32, "f64": np.float64, "wide": np.float64, "mixed": np.float64}


def values(kind, nnz, nx, ny, seed):
    """int64 (a, x, y0) for a matrix of nnz stored entries, x of nx and y of ny entries"""
    rng = np.random.default_rng(seed)
    (alo, ahi), (xlo, xhi), (ylo, yhi) = _RANGES[kind]
    a = nonzero_ints(rng, nnz, alo, ahi)
    x = nonzero_ints(rng, nx, xlo, xhi)
    y0 = 2 * rng.integers(-yhi + 1, yhi, ny, dtype=np.int64) if yhi > 1 else np.zeros(ny, np.int64)
    return a, x, y0


# ------------------------------------------------------------------------------------------------ structure
def lens_to_structure(lens, cols, seed):
    """Row offsets and distinct, sorted columns per row for the given row lengths (every length <= cols)."""
    lens = np.asarray(lens, np.int64)
    assert lens.size == 0 or lens.max() <= cols
    rng = np.random.default_rng(seed)
    off = np.concatenate([[0], np.cumsum(lens)]).astype(np.int32)
    parts = []
    for l in lens:
        l = int(l)
        if l == 0:
            continue
        if l > cols // 8:
            c = rng.choice(cols, size=l, replace=False)
        else:
            c = np.unique(rng.integers(0, cols, size=2 * l + 8))
            while c.size < l:
                c = np.unique(np.concatenate([c, rng.integers(0, cols, size=2 * l + 8)]))
            c = rng.permutation(c)[:l]
        parts.append(np.sort(c))
    col = (np.concatenate(parts) if parts else np.zeros(0, np.int64)).astype(np.int32)
    return off, col


class Fixture:
    """One exact SpMV problem: structure (off, col: int32, base 0), int64 values a / x / y0, and their float views."""

    def __init__(self, name, lens, cols, kind, seed=0):
        self.name, self.kind, self.cols = name, kind, int(cols)
        self.off, self.col = lens_to_structure(lens, cols, seed)
        self.rows, self.nnz = self.off.size - 1, int(self.off[-1])
        self.a, self.x, self.y0 = values(kind, self.nnz, self.cols, self.rows, seed + 1)
        _, self.xt, self.y0t = values(kind, 0, self.rows, self.cols, seed + 2)         # A^T: x[rows], y[cols]
        self.p = MANTISSA[kind]

    @property
    def val(self):
        return self.a.astype(NP_A[self.kind])

    def xf(self, transpose=False):
        return (self.xt if transpose else self.x).astype(NP_XY[self.kind])

    def y0f(self, transpose=False):
        return (self.y0t if transpose else self.y0).astype(NP_XY[self.kind])

    def want(self, alpha, beta, transpose=False):
        x, y0 = (self.xt, self.y0t) if transpose else (self.x, self.y0)
        return reference(self.off, self.col, self.a, x, y0, alpha, beta, transpose=transpose, cols=self.cols)

    def check(self, alpha, beta, transpose=False):
        x, y0 = (self.xt, self.y0t) if transpose else (self.x, self.y0)
        check_exact(self.off, self.col, self.a, x, y0, alpha, beta, self.p, transpose=transpose, cols=self.cols)


# ------------------------------------------------------------------------------------------------ the reference
def _twice(s):
    t = 2 * s
    assert t == int(t), f"{s}: alpha / beta must be multiples of 1/2"
    return int(t)


def row_sums(off, col, a, x, transpose=False, cols=None, absolute=False):
    """S[r] = sum_k a[k] * x[col[k]] over row r (A^T: S[c] = sum over column c of a * x[row]) in int64"""
    off = np.asarray(off, np.int64)
    rows = off.size - 1
    row = np.repeat(np.arange(rows), np.diff(off))
    col = np.asarray(col, np.int64)
    p = a * (x[row] if transpose else x[col])
    if absolute:
        p = np.abs(p)
    out = np.zeros(cols if transpose else rows, np.int64)
    np.add.at(out, col if transpose else row, p)
    return out


def reference(off, col, a, x, y0, alpha, beta, transpose=False, cols=None):
    """alpha * A x + beta * y0 from integers (beta == 0: y0 is not read), returned as float64 (exact: a multiple of 1/2)"""
    s = row_sums(off, col, a, x, transpose, cols)
    num = _twice(alpha) * s
    if beta != 0:
        num = num + _twice(beta) * np.asarray(y0, np.int64)
    assert np.all(np.abs(num) < (1 << 53))
    return num.astype(np.float64) / 2


def check_exact(off, col, a, x, y0, alpha, beta, p, transpose=False, cols=None):
    """The exactness precondition, per row: sum |products| < 2^p and 2 * (|alpha| sum |products| + |beta y0|) < 2^p.  Then
    every partial sum of the row (any order, any split) and the result itself are exact in a p-bit significand."""
    s = row_sums(off, col, a, x, transpose, cols, absolute=True)
    bound = abs(_twice(alpha)) * s
    if beta != 0:
        bound = bound + abs(_twice(beta)) * np.abs(np.asarray(y0, np.int64))
    limit = 1 << p
    assert np.all(s < limit), f"row sum of |products| reaches 2^{p}"
    assert np.all(bound < limit), f"|result| reaches 2^{p - 1}"
    assert np.all(np.asarray(a) != 0) and np.all(np.asarray(x) != 0), "a zero value hides a dropped product"


def spmm_reference(off, col, a, B, C0, alpha, beta):
    """alpha * A B + beta * C0 with B (cols x n) / C0 (rows x n) int64 2-D arrays; float64, exact"""
    off = np.asarray(off, np.int64)
    rows = off.size - 1
    row = np.repeat(np.arange(rows), np.diff(off))
    S = np.zeros((rows, B.shape[1]), np.int64)
    np.add.at(S, row, a[:, None] * B[np.asarray(col, np.int64)])
    num = _twice(alpha) * S + (_twice(beta) * C0 if beta != 0 else 0)
    return np.asarray(num, np.float64) / 2


def to_sell(off, col, val, S, base=0, min_width=None, pad_val=0.0):
    """Sliced-ELL (slice-column-major, padding column -1 + base) of a base-0 CSR; min_width: {slice: width} to widen slices
    with padding beyond their longest row (width > 0 on a slice of empty rows = a slice of padding only); pad_val: the value
    stored in the padding slots."""
    off = np.asarray(off, np.int64)
    rows = off.size - 1
    ns = (rows + S - 1) // S
    lens = np.diff(off)
    so = [0]
    for s in range(ns):
        w = int(lens[s * S:(s + 1) * S].max()) if rows else 0
        w = max(w, (min_width or {}).get(s, 0))
        so.append(so[-1] + w * S)
    sc = np.full(so[-1], -1 + base, np.int32)
    sv = np.full(so[-1], pad_val, np.asarray(val).dtype)
    for r in range(rows):
        s, i = divmod(r, S)
        for k in range(int(lens[r])):
            sc[so[s] + k * S + i] = col[off[r] + k] + base
            sv[so[s] + k * S + i] = val[off[r] + k]
    return np.asarray(so, np.int32) + base, sc, sv          # slice offsets carry the index base like the columns


def check_spmm_exact(off, col, a, B, C0, p):
    """check_exact for C = alpha A B + beta C0, every (alpha, beta) of SCALARS at once"""
    amax = max(abs(_twice(al)) for al, _ in SCALARS)
    bmax = max(abs(_twice(be)) for _, be in SCALARS)
    s = spmm_reference(off, col, np.abs(a), np.abs(B), np.abs(C0), 0.5, 0.0)        # sum |products| per entry of C
    assert np.all(s < (1 << p)) and np.all(amax * s + bmax * np.abs(C0) < (1 << p))
    assert np.all(a != 0) and np.all(B != 0)


# ------------------------------------------------------------------------------------------------ boundary profiles
def ends_at(positions):
    """row lengths whose rows end (exclusive end = off[r + 1]) at the given non-decreasing non-zero positions; a repeated
    position makes empty rows"""
    pos = np.asarray(positions, np.int64)
    assert np.all(np.diff(pos) >= 0)
    return np.diff(np.concatenate([[0], pos]))


def _block_of(total, n=32):
    """n row lengths summing to `total`, as even as possible (one block of csr_short_kernel)"""
    q, r = divmod(total, n)
    return [q + 1] * r + [q] * (n - r)


def boundary_profiles(P: dict) -> dict:
    """name -> (row lengths, cols).  P = kernel_params()."""
    W, CT, T, L, CAP = P["warp_chunk"], P["cta_nnz"], P["tile"], P["long_row"], P["short_cap"]
    prof = {}
    # row ends at lane 0 and lane 31 of a 32-wide step, and more than 32 row ends inside one warp chunk
    prof["lane_ends"] = ([1] + [32] * 12 + [31, 1, 33, 63, 1] + [1] * 40 + [0, 0] + [2] * 20, 4096)
    # row ends at border - 1, border, border + 1 of every warp chunk and every CTA, with runs of empty rows on the borders
    pos = []
    for k in range(1, 8):
        pos += [k * W - 1, k * W, k * W + 1] if k % 2 else [k * W, k * W, k * W]          # even k: empty rows on the border
    for k in range(1, 6):
        base = 2 * k * CT
        pos += [base - 1, base, base + 1] + ([base + W] * 3 if k % 2 else [])
    pos += [pos[-1] + 5]
    prof["chunk_and_cta_borders"] = (ends_at(pos), 8192)
    # tile borders (merge path: row ends + non-zeros, rows of at least LONG_ROW are cut) and rows around LONG_ROW
    prof["long_row_edges"] = ([L - 1, L, L + 1] * 6 + [3, 0, 0, L + 1, L - 1, 0, L], 8192)
    prof["tile_border_ends"] = ([T - 1 - 1, T - 1, T - 1 + 1, T - 2, T - 3, 1, T - 1, 0, T - 1, T + 1] * 2, 8192)
    # rows crossing exactly 1, 2 and >= 3 CTA / tile borders
    prof["rows_cross_borders"] = ([5, CT, 3, 2 * CT + 7, 0, 1, 3 * CT + 11, 2, T + 9, 0, 4 * T + 1, 6], 16384)
    # 32-row blocks of csr_short_kernel with CAP - 1, CAP, CAP + 1 and 2 * CAP non-zeros
    lens = []
    for tot in (CAP - 1, CAP, CAP + 1, 2 * CAP, 7, 0, CAP + 1, CAP - 1):
        lens += _block_of(tot)
    prof["short_block_caps"] = (lens + [3, 0, 5], 4096)
    # leading and trailing empty rows, empty runs inside
    prof["leading_trailing_empty"] = ([0] * 37 + [W - 1, 1, 0, 0, 0, CT - W, 0, 0, 5] + [0] * 45, 4096)
    # degenerate shapes
    prof["nnz_zero"] = ([0] * 70, 50)
    prof["one_row"] = ([37], 64)
    prof["one_col"] = ([1] * 40 + [0, 1], 1)
    prof["rect_tall"] = (list(np.random.default_rng(3).integers(0, 8, 300)), 17)
    prof["rect_wide"] = (list(np.random.default_rng(4).integers(0, 700, 40)), 3000)
    # seeded random mixes of all of the above
    for seed in range(3):
        rng = np.random.default_rng(1000 + seed)
        n = int(rng.integers(150, 400))
        kind = rng.integers(0, 6, n)
        lens = np.where(kind == 0, 0, np.where(kind == 1, rng.integers(1, 6, n), np.where(kind == 2, rng.integers(6, 80, n),
                        np.where(kind == 3, rng.integers(L - 2, L + 3, n), np.where(kind == 4, rng.integers(W - 2, W + 3, n),
                                                                                      rng.integers(CT - 2, 3 * CT, n))))))
        prof[f"random_mix_{seed}"] = (list(lens), 8192)
    return {k: (np.asarray(v, np.int64), c) for k, (v, c) in prof.items()}


BOUNDARY_CLASSES = (
    ["end_lane0", "end_lane31", "more_than_32_ends_in_a_warp_chunk", "long_row_minus1", "long_row", "long_row_plus1",
     "leading_empty", "trailing_empty", "nnz_zero", "one_row", "one_col", "rectangular"]
    + [f"end_{b}_{d}" for b in ("warp_chunk", "cta", "tile") for d in ("m1", "0", "p1")]
    + [f"cross_{b}_{k}" for b in ("cta", "tile") for k in ("1", "2", "3+")]
    + [f"empty_run_on_{b}" for b in ("warp_chunk", "cta")]
    + [f"short_block_{t}" for t in ("cap_m1", "cap", "cap_p1", "2cap")]
)


def coverage(off, cols, P: dict) -> set:
    """Which of BOUNDARY_CLASSES this matrix hits, recomputed from its row offsets (base 0)."""
    from oracle.partition_ref import csr_partition
    off = np.asarray(off, np.int64)
    rows, nnz = off.size - 1, int(off[-1])
    lens = np.diff(off)
    hit = set()
    if nnz == 0:
        hit.add("nnz_zero")
    if rows == 1:
        hit.add("one_row")
    if cols == 1:
        hit.add("one_col")
    if rows != cols:
        hit.add("rectangular")
    if rows and lens[0] == 0 and nnz:
        hit.add("leading_empty")
    if rows and lens[-1] == 0 and nnz:
        hit.add("trailing_empty")
    ne = lens > 0
    end = off[1:][ne]                           # exclusive end of every non-empty row
    last = end - 1                              # its last non-zero
    if np.any(last % 32 == 0):
        hit.add("end_lane0")
    if np.any(last % 32 == 31):
        hit.add("end_lane31")
    if last.size and np.bincount(last // P["warp_chunk"]).max() > 32:
        hit.add("more_than_32_ends_in_a_warp_chunk")
    L = P["long_row"]
    for name, n in (("long_row_minus1", L - 1), ("long_row", L), ("long_row_plus1", L + 1)):
        if np.any(lens == n):
            hit.add(name)
    for b, B in (("warp_chunk", P["warp_chunk"]), ("cta", P["cta_nnz"])):
        inner = end[(end >= B) & (end < nnz)] if nnz else end[:0]
        for d, dd in (("m1", -1), ("0", 0), ("p1", 1)):
            if np.any((inner - dd) % B == 0):
                hit.add(f"end_{b}_{d}")
        empty_at = off[:-1][~ne]
        if np.any((empty_at > 0) & (empty_at < nnz) & (empty_at % B == 0) & np.r_[False, ~ne[:-1]][~ne]):
            hit.add(f"empty_run_on_{b}")           # two or more empty rows in a row, sitting on the border
    if nnz:
        # CTA borders: multiples k * cta_nnz with off[r] < k * cta_nnz < off[r + 1]
        CT = P["cta_nnz"]
        inside = np.where(ne, (off[1:] - 1) // CT - off[:-1] // CT, 0)
        for k, name in ((1, "1"), (2, "2")):
            if np.any(inside == k):
                hit.add(f"cross_cta_{name}")
        if np.any(inside >= 3):
            hit.add("cross_cta_3+")
        # tile borders: the merge-path partition of the tile kernels (row ends + non-zeros; long rows cut at the diagonal)
        tiles = csr_partition(off, 0, P["tile"], L).astype(np.int64)
        tn = tiles[1:-1, 1]
        cuts = np.zeros(rows, np.int64)
        r_of = np.searchsorted(off, tn, side="right") - 1          # row holding non-zero tn
        strictly = (tn > off[np.minimum(r_of, rows)]) & (r_of < rows)
        np.add.at(cuts, r_of[strictly], 1)
        for k, name in ((1, "1"), (2, "2")):
            if np.any(cuts == k):
                hit.add(f"cross_tile_{name}")
        if np.any(cuts >= 3):
            hit.add("cross_tile_3+")
        d = np.arange(1, tiles.shape[0] - 1) * P["tile"]
        g_end = np.arange(1, rows + 1)[ne] + end                   # merge position right after each row end
        for dname, dd in (("m1", -1), ("0", 0), ("p1", 1)):
            if np.intersect1d(g_end - dd, d).size:
                hit.add(f"end_tile_{dname}")
    # 32-row blocks of csr_short_kernel
    R, CAP = P["short_rows"], P["short_cap"]
    tot = np.diff(off[np.minimum(np.arange(0, rows + R, R), rows)])     # non-zeros per block (the last one may be partial)
    for name, t in (("cap_m1", CAP - 1), ("cap", CAP), ("cap_p1", CAP + 1), ("2cap", 2 * CAP)):
        if np.any(tot == t):
            hit.add(f"short_block_{name}")
    return hit


# ------------------------------------------------------------------------------------------------ fused CG BLAS-1 (cg_fused.cu)
def cg_params(lib=None) -> dict:
    """block (threads per CTA) and max_ctas (grid cap) of the built library's CG kernels (b200cg_params)"""
    if lib is None:
        from cudalibrarysamples_b200 import lib as _lib
        lib = _lib.shim()
    b, m = C.c_int32(), C.c_int32()
    lib.b200cg_params(C.byref(b), C.byref(m))
    return dict(block=b.value, max_ctas=m.value)


def cg_grid(n, P):
    """CTAs of a launch over n elements (grid_for in cg_fused.cu: one pair per thread, capped)"""
    g = (n // 2 + P["block"] - 1) // P["block"]
    return int(max(1, min(g, P["max_ctas"])))


def cg_walk(n, P):
    """The index walk every kernel of cg_fused.cu makes: thread k of the grid starts at pair index 2k and strides by
    2 * grid * block; i + 1 < n takes the 16-byte path (elements i, i + 1), otherwise the scalar path (element i).
    Returns grid, passes (grid-stride trips of thread 0), visits[i] (how often element i is read) and the trip on which the
    scalar path ran (None if it never did)."""
    g = cg_grid(n, P)
    first = 2 * np.arange(g * P["block"], dtype=np.int64)
    stride = 2 * g * P["block"]
    visits = np.zeros(n, np.int64)
    passes, scalar_pass, scalar_visits = 0, None, 0
    while True:
        i = first + passes * stride
        i = i[i < n]
        if i.size == 0:
            break
        pair, single = i[i + 1 < n], i[i + 1 >= n]
        visits[pair] += 1
        visits[pair + 1] += 1
        visits[single] += 1
        if single.size:
            scalar_pass, scalar_visits = passes, scalar_visits + single.size
        passes += 1
    return dict(grid=g, passes=passes, visits=visits, scalar_pass=scalar_pass, scalar_visits=scalar_visits)


def cg_full_pass(P):
    """F: elements one grid-stride pass covers at the grid cap"""
    return P["max_ctas"] * 2 * P["block"]


def cg_sizes(P):
    """Vector lengths around the kernels' borders: P2 = 2 * block elements per CTA pass, F per full-grid pass"""
    P2, F = 2 * P["block"], cg_full_pass(P)
    first_at_cap = 2 * ((P["max_ctas"] - 1) * P["block"] + 1)          # smallest n with cg_grid(n) == max_ctas
    return [0, 1, 2, 3, 33, P2 - 1, P2, P2 + 1, 2 * P2 + 1, 5 * P2 + 1, first_at_cap, F - 1, F, F + 1, F + 2, 2 * F, 2 * F + 3,
            3 * F + P2 + 1]


CG_CLASSES = ["n_zero", "scalar_tail_only", "odd_tail_first_pass", "odd_tail_later_pass_below_cap", "odd_tail_later_pass_at_cap",
              "one_cta", "two_ctas", "cap_single_pass", "exactly_one_full_pass", "multi_pass_partial_last",
              "multi_pass_whole_passes"]


def cg_coverage(n, P) -> set:
    """Which of CG_CLASSES a launch over n elements falls in, from the index model"""
    w = cg_walk(n, P)
    F, cap = cg_full_pass(P), w["grid"] == P["max_ctas"]
    sp = w["scalar_pass"]
    hit = set()
    if n == 0:
        return {"n_zero"}
    if n == 1:
        hit.add("scalar_tail_only")
    elif sp == 0:
        hit.add("odd_tail_first_pass")
    if sp is not None and sp > 0:
        hit.add("odd_tail_later_pass_at_cap" if cap else "odd_tail_later_pass_below_cap")
    if w["grid"] in (1, 2):
        hit.add("one_cta" if w["grid"] == 1 else "two_ctas")
    if cap and w["passes"] == 1:
        hit.add("cap_single_pass")
    if n == F:
        hit.add("exactly_one_full_pass")
    if w["passes"] > 1 and cap:
        hit.add("multi_pass_whole_passes" if n % F == 0 else "multi_pass_partial_last")
    return hit


CG_KINDS = ["f64", "wide"]
_CG_RANGES = {"f64": (1, 5), "wide": (1 << 12, 1 << 13)}      # |value|: products of "wide" need 25-26 bits, sums far more than fp32 has
# the device scalars: alpha = delta / denom = -1/4 and beta = delta_new / delta = 1/2, both exact divisions
CG_SCALARS = dict(delta=3.0, denom=-12.0, delta_new=1.5)


class CgKernel:
    """One entry point: its vector arguments and device-scalar arguments in call order (the workspace comes last when
    `workspace`), the vectors it writes and the scalar it reduces into (None: no reduction)."""

    def __init__(self, vectors, scalars, writes, reduces, workspace):
        self.vectors, self.scalars, self.writes, self.reduces, self.workspace = vectors, scalars, writes, reduces, workspace


CG_KERNELS = {
    "dot": CgKernel(["a", "b"], ["out"], [], "out", True),
    "update_r": CgKernel(["r", "t"], ["delta", "denom", "delta_new"], ["r"], "delta_new", True),
    "update_xr": CgKernel(["x", "r", "p", "t"], ["delta", "denom", "delta_new"], ["x", "r"], "delta_new", True),
    "update_xp": CgKernel(["x", "p", "r"], ["delta", "denom", "delta_new"], ["x", "p"], None, False),
    "update_p": CgKernel(["p", "r"], ["delta_new", "delta"], ["p"], None, False),
}


def cg_vectors(kind, n, names, seed):
    """int64 vectors of n nonzero integers each (|v| in the kind's range), one per name"""
    rng = np.random.default_rng(seed)
    lo, hi = _CG_RANGES[kind]
    return {k: nonzero_ints(rng, n, lo, hi) for k in names}


def _dyadic(q: Fraction):
    assert q.denominator & (q.denominator - 1) == 0, f"{q}: not a dyadic quotient"
    return q.numerator, q.denominator


def _exact_float(num, den):
    """num / den as float64, asserting that it is exact (|num| < 2^53, den a power of two)"""
    assert np.all(np.abs(num) < (1 << 53)), "a result needs more than 53 bits"
    return np.asarray(num, np.int64).astype(np.float64) / den


def cg_reference(name, v, scal=CG_SCALARS):
    """What kernel `name` must produce from the int64 vectors v (dict) and the device scalars: {written vector or reduced
    scalar: float64}, computed in integers.  Asserts the exactness precondition: every updated element is num / 4 with
    |num| < 2^53, and the sum of |terms| of each reduction stays below 2^53 in units of its last place (1 for a . b, 1/16 for
    r . r), so every partial sum in any order is exact."""
    alpha = Fraction(scal["delta"]) / Fraction(scal["denom"])
    beta = Fraction(scal["delta_new"]) / Fraction(scal["delta"])
    an, ad = _dyadic(alpha)
    bn, bd = _dyadic(beta)
    out = {}
    if name == "dot":
        terms = v["a"] * v["b"]
        assert int(np.abs(terms).sum()) < (1 << 53)
        out["out"] = float(int(terms.sum()))
    if name in ("update_r", "update_xr"):
        rn = v["r"] * ad - an * v["t"]                       # r - alpha t, scaled by ad
        sq = rn * rn
        assert int(sq.sum()) < (1 << 53)
        out["r"] = _exact_float(rn, ad)
        out["delta_new"] = float(int(sq.sum())) / (ad * ad)
    if name in ("update_xr", "update_xp"):
        out["x"] = _exact_float(v["x"] * ad + an * v["p"], ad)      # x + alpha p
    if name in ("update_xp", "update_p"):
        out["p"] = _exact_float(v["r"] * bd + bn * v["p"], bd)      # r + beta p
    return out
