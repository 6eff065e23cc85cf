"""numpy restatement of the native SpGEMM numeric phase (b200spgemm_compute, DESIGN.md 3.28).

For every stored C(i, j) of a given C pattern: acc = +0, then for each stored (i, k) of A in A's stored order and the stored (k, j)
of B, acc = fl(acc + fl(a_ik * b_kj)); then C(i, j) = fl(fl(alpha * acc) + fl(beta * c_ij)), or fl(alpha * acc) at beta = 0 (C is
not read).  Every operation is one correctly rounded IEEE operation of the value type (numpy float32 / float64 scalars round each
operation), so the result is the kernel's bit for bit.  The fold is vectorised over the entries of one C row: their accumulations
are independent, and each entry still sees its products in A's order.

Also the pattern helpers the tests and scripts/spgemm_bench.py share: CSR arrays of the structural product (every (i, j) some
a_ik b_kj reaches, values or not), the workloads and their traffic and product counts."""
from __future__ import annotations

import numpy as np
import scipy.sparse as sp


def structural_pattern(a_off, a_col, b_off, b_col, rows, cols):
    """(off, col) of the pattern of A B: every (i, j) with a stored a_ik and b_kj, columns ascending (what the closed reuse_nnz
    builds, pinned on the H100)."""
    A = sp.csr_matrix((np.ones(len(a_col)), np.asarray(a_col), np.asarray(a_off)), shape=(rows, len(b_off) - 1))
    B = sp.csr_matrix((np.ones(len(b_col)), np.asarray(b_col), np.asarray(b_off)), shape=(len(b_off) - 1, cols))
    P = (A @ B).tocsr()
    P.sort_indices()
    return P.indptr.astype(np.int32), P.indices.astype(np.int32)


def spgemm(a_off, a_col, a_val, b_off, b_col, b_val, c_off, c_col, c_val=None, alpha=1.0, beta=0.0):
    """C's values on (c_off, c_col) (base 0 arrays; columns ascending per row) as b200spgemm_compute computes them, in the dtype of
    a_val.  A product whose column C's row does not store is skipped."""
    dt = np.asarray(a_val).dtype.type
    a_off, a_col, a_val = np.asarray(a_off), np.asarray(a_col), np.asarray(a_val)
    b_off, b_col, b_val = np.asarray(b_off), np.asarray(b_col), np.asarray(b_val)
    c_off, c_col = np.asarray(c_off), np.asarray(c_col)
    out = np.empty(len(c_col), dtype=dt)
    for i in range(len(c_off) - 1):
        c0, c1 = int(c_off[i]), int(c_off[i + 1])
        cols = c_col[c0:c1]
        acc = np.zeros(c1 - c0, dtype=dt)
        for p in range(int(a_off[i]), int(a_off[i + 1])):
            k = int(a_col[p])
            bs = slice(int(b_off[k]), int(b_off[k + 1]))
            j = b_col[bs]
            pos = np.searchsorted(cols, j)
            hit = pos < len(cols)
            hit[hit] = cols[pos[hit]] == j[hit]
            prod = (dt(a_val[p]) * b_val[bs][hit]).astype(dt)          # one rounding per product
            acc[pos[hit]] = (acc[pos[hit]] + prod).astype(dt)          # distinct columns in a B row: one add per slot
        v = (dt(alpha) * acc).astype(dt)
        if beta != 0:
            v = (v + (dt(beta) * np.asarray(c_val[c0:c1], dtype=dt)).astype(dt)).astype(dt)
        out[c0:c1] = v
    return out


def spgemm_loop(a_off, a_col, a_val, b_off, b_col, b_val, c_off, c_col, c_val=None, alpha=1.0, beta=0.0):
    """The same fold written entry by entry with Python scalars of the value type: the plain statement spgemm() is checked against."""
    dt = np.asarray(a_val).dtype.type
    out = np.empty(len(c_col), dtype=dt)
    for i in range(len(c_off) - 1):
        for p in range(int(c_off[i]), int(c_off[i + 1])):
            j = int(c_col[p])
            acc = dt(0)
            for q in range(int(a_off[i]), int(a_off[i + 1])):
                k = int(a_col[q])
                for e in range(int(b_off[k]), int(b_off[k + 1])):
                    if int(b_col[e]) == j:
                        acc = dt(acc + dt(dt(a_val[q]) * dt(b_val[e])))
            v = dt(dt(alpha) * acc)
            out[p] = v if beta == 0 else dt(v + dt(dt(beta) * dt(c_val[p])))
    return out


# ---- workloads ---------------------------------------------------------------------------------------------------------------
def stencil5(n):
    """5-point Laplacian on an n x n grid (4 on the diagonal, -1 off it), CSR (off, col, val float64)."""
    I = sp.identity(n, format="csr")
    T = sp.diags([-1.0, 2.0, -1.0], [-1, 0, 1], shape=(n, n), format="csr")
    M = (sp.kron(I, T) + sp.kron(T, I)).tocsr()
    M.sort_indices()
    return M.indptr.astype(np.int32), M.indices.astype(np.int32), M.data.astype(np.float64)


def stencil7(n):
    """7-point Laplacian on an n x n x n grid, CSR."""
    I = sp.identity(n, format="csr")
    T = sp.diags([-1.0, 2.0, -1.0], [-1, 0, 1], shape=(n, n), format="csr")
    M = (sp.kron(sp.kron(I, I), T) + sp.kron(sp.kron(I, T), I) + sp.kron(sp.kron(T, I), I)).tocsr()
    M.sort_indices()
    return M.indptr.astype(np.int32), M.indices.astype(np.int32), M.data.astype(np.float64)


def restriction2(n):
    """2:1 aggregation restriction of an n x n grid (n even): row (I, J) of the (n/2)^2 coarse points sums the four fine points
    (2I + a, 2J + b), a, b in {0, 1}, with weight 1/4.  ((n/2)^2 x n^2 CSR)"""
    m = n // 2
    I, J = np.meshgrid(np.arange(m), np.arange(m), indexing="ij")
    rows = np.repeat((I * m + J).ravel(), 4)
    fine = np.stack([(2 * I + a) * n + 2 * J + b for a in (0, 1) for b in (0, 1)], axis=-1).reshape(-1)
    R = sp.csr_matrix((np.full(len(rows), 0.25), (rows, fine)), shape=(m * m, n * n))
    R.sort_indices()
    return R.indptr.astype(np.int32), R.indices.astype(np.int32), R.data.astype(np.float64)


def uniform(n, per_row, seed):
    """n x n with per_row uniformly random columns in every row (a repeated column merged), ascending, values in [-1, 1)."""
    rng = np.random.default_rng(seed)
    M = sp.csr_matrix((rng.uniform(-1, 1, n * per_row), (np.repeat(np.arange(n), per_row), rng.integers(0, n, n * per_row))),
                      shape=(n, n))
    M.sum_duplicates()
    M.sort_indices()
    return M.indptr.astype(np.int32), M.indices.astype(np.int32), M.data.astype(np.float64)


def rmat(scale, per_row, seed, a=0.57, b=0.19, c=0.19):
    """R-MAT 2^scale x 2^scale with about per_row entries per row (duplicates merged), CSR with ascending columns."""
    rng = np.random.default_rng(seed)
    n, m = 1 << scale, per_row << scale
    r = np.zeros(m, np.int64)
    q = np.zeros(m, np.int64)
    for _ in range(scale):
        u = rng.random(m)
        down = u >= a + b
        right = ((u >= a) & (u < a + b)) | (u >= a + b + c)
        r = 2 * r + down
        q = 2 * q + right
    M = sp.csr_matrix((rng.uniform(-1, 1, m), (r, q)), shape=(n, n))
    M.sum_duplicates()
    M.sort_indices()
    return M.indptr.astype(np.int32), M.indices.astype(np.int32), M.data.astype(np.float64)


def products_per_row(a_off, a_col, b_off):
    """Products of every C row: sum over A row i's k of nnz(B row k), int64."""
    blen = np.diff(np.asarray(b_off, dtype=np.int64))
    per = blen[np.asarray(a_col)]
    cs = np.concatenate([[0], np.cumsum(per)])
    a_off = np.asarray(a_off, dtype=np.int64)
    return cs[a_off[1:]] - cs[a_off[:-1]]


def traffic_bytes(rows, nnz_a, nnz_b, nnz_c, products, value_bytes):
    """Least bytes one numeric pass moves: A, C's pattern read and C's values written once, and one B entry (column and value) per
    product, with B's offsets read per A entry."""
    return (rows + 1) * 4 * 2 + nnz_a * (8 + value_bytes) + nnz_c * (4 + value_bytes) + products * (4 + value_bytes)
