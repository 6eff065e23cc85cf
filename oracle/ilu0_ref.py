"""Numpy restatement of the incomplete factorizations without fill-in of csrc/ilu0_csr.cu (cusparse<t>csrilu02 / csric02).

The pattern is CSR with columns strictly ascending in every row and a stored diagonal in every row.  Every operation is one
correctly rounded multiply, subtract, divide or square root in the value type (numpy's float32 / float64 ufuncs, never fused),
and every entry is a left fold in ascending column order: the bits below are the kernel's, whatever its schedule.

- ILU(0), row form (IKJ): for each stored (i, k), k < i, ascending: a_ik <- a_ik / a_kk, then a_ij <- a_ij - a_ik a_kj for every
  stored (k, j), j > k, that row i also stores.  Then the pivot's boost (|a_ii| <= tol -> boost_val) and zero check.
- IC(0), lower triangle only: for each stored (i, k), k < i, ascending: l_ik <- a_ik / l_kk; a_ij <- a_ij - l_ik l_jk for every
  stored (i, j), k < j < i, with (j, k) stored; a_ii <- a_ii - l_ik l_ik.  Then l_ii <- sqrt(a_ii).  Entries with j > i are
  untouched.

Rows are processed level by level (a row's level is 1 + the largest level of the rows its strictly-lower entries name), and within a
level step by step, vectorised over the level's rows: rows of one level never read each other, so this is the sequential order's
result.  The textbook dense loops (dense_ilu0 / dense_ic0) check this restatement on small matrices.
"""
from __future__ import annotations

import numpy as np

INT32_MAX = 2**31 - 1


def _pattern(off, col, base):
    off = np.asarray(off, np.int64) - base
    col = np.asarray(col, np.int64) - base
    n = off.size - 1
    rowof = np.repeat(np.arange(n), np.diff(off))
    return off, col, n, rowof


def diag_positions(off, col, base=0):
    """Position of each row's diagonal (-1 where a row stores none)."""
    off, col, n, rowof = _pattern(off, col, base)
    d = np.full(n, -1, np.int64)
    hit = np.nonzero(col == rowof)[0]
    d[rowof[hit]] = hit
    return d


def pattern_ok(off, col, base=0):
    """Columns strictly ascending and in range in every row."""
    off, col, n, rowof = _pattern(off, col, base)
    if np.any(col < 0) or np.any(col >= n):
        return False
    same = rowof[1:] == rowof[:-1]
    return not np.any(same & (np.diff(col) <= 0))


def levels(off, col, base=0):
    """Level of every row of the strictly-lower dependency graph."""
    off, col, n, rowof = _pattern(off, col, base)
    lev = np.zeros(n, np.int64)
    lower = col < rowof
    lo_off = np.concatenate([[0], np.cumsum(np.bincount(rowof[lower], minlength=n))])
    lo_col = col[lower].tolist()
    lv = [0] * n
    for i in range(n):
        m = 0
        for p in range(lo_off[i], lo_off[i + 1]):
            v = lv[lo_col[p]] + 1
            if v > m:
                m = v
        lv[i] = m
    lev[:] = lv
    return lev


def _find(key, targets):
    """Positions of targets in the sorted key array, -1 where absent."""
    pos = np.searchsorted(key, targets)
    pos = np.minimum(pos, key.size - 1)
    return np.where(key[pos] == targets, pos, -1)


def factor(kind, off, col, val, base=0, boost=False, tol=0.0, boost_val=0.0):
    """The factor of kind "lu" / "ic" of the CSR matrix, in val's dtype: (new values, zero-pivot row or -1).  The zero-pivot row is the
    smallest row whose pivot is zero (LU, after the boost) or not positive (IC, before its square root), or without a stored diagonal
    (a structural zero).  Such a row is left as stored, and nothing is read from it: a step whose row k has no diagonal is skipped,
    as an IC update whose l_jk lies in such a row is."""
    T = np.asarray(val).dtype.type
    a = np.array(val, dtype=T, copy=True)
    offz, colz, n, rowof = _pattern(off, col, base)
    d = diag_positions(off, col, base)
    if not pattern_ok(off, col, base):
        raise ValueError("unsorted, duplicate or out-of-range columns")
    key = rowof * n + colz                           # ascending: rows in order, columns ascending within a row
    nlower = d - offz[:-1]                           # strictly-lower entries per row (they come first)
    lev = levels(off, col, base)
    order = np.argsort(lev, kind="stable")
    bounds = np.searchsorted(lev[order], np.arange(lev.max() + 2 if n else 1))
    for l in range(len(bounds) - 1):
        rows = order[bounds[l]:bounds[l + 1]]
        rows = rows[d[rows] >= 0]
        for s in range(int(nlower[rows].max()) if rows.size else 0):
            r = rows[nlower[rows] > s]
            p = offz[r] + s                          # entry (i, k) of this step
            has = d[colz[p]] >= 0
            r, p = r[has], p[has]
            k = colz[p]
            with np.errstate(divide="ignore", invalid="ignore"):     # after a zero pivot, as on the device
                lik = a[p] / a[d[k]]
            a[p] = lik
            if kind == "lu":
                # every stored (k, j), j > k: a_ij -= l_ik a_kj where row i stores j
                cnt = offz[k + 1] - (d[k] + 1)
                rr = np.repeat(np.arange(r.size), cnt)
                q = np.repeat(d[k] + 1 - np.cumsum(np.concatenate([[0], cnt[:-1]])), cnt) + np.arange(cnt.sum())
                tgt = _find(key, r[rr] * n + colz[q])
                ok = tgt >= 0
                a[tgt[ok]] = a[tgt[ok]] - lik[rr[ok]] * a[q[ok]]
            else:
                # every stored (i, j), k < j < i: a_ij -= l_ik l_jk where row j stores k
                cnt = d[r] - (p + 1)
                rr = np.repeat(np.arange(r.size), cnt)
                q = np.repeat(p + 1 - np.cumsum(np.concatenate([[0], cnt[:-1]])), cnt) + np.arange(cnt.sum())
                src = _find(key, colz[q] * n + k[rr])
                ok = (src >= 0) & (d[colz[q]] >= 0)
                a[q[ok]] = a[q[ok]] - lik[rr[ok]] * a[src[ok]]
                a[d[r]] = a[d[r]] - lik * lik
        if kind == "lu":
            piv = a[d[rows]]
            if boost:
                small = np.abs(piv.astype(np.float64)) <= tol
                a[d[rows[small]]] = T(boost_val)
        else:
            piv = a[d[rows]]
            with np.errstate(invalid="ignore"):
                a[d[rows]] = np.sqrt(piv)
    # LU: the pivot after its boost.  IC: sqrt is exact at 0 and NaN below it, so l_ii > 0 exactly where its argument was.
    piv = np.ones(n, T)
    piv[d >= 0] = a[d[d >= 0]]
    bad = np.nonzero((d < 0) | ((piv == 0) if kind == "lu" else ~(piv > 0)))[0]
    return a, (int(bad[0]) if bad.size else -1)


# ---------------------------------------------------------------------------------------------------- textbook loops
def dense_ilu0(A):
    """ILU(0) of a dense matrix on its non-zero pattern (IKJ), in A's dtype: L and U overwrite A."""
    A = np.array(A, copy=True)
    n = A.shape[0]
    S = A != 0
    for i in range(1, n):
        for k in range(i):
            if not S[i, k]:
                continue
            A[i, k] = A[i, k] / A[k, k]
            for j in range(k + 1, n):
                if S[i, j] and S[k, j]:
                    A[i, j] = A[i, j] - A[i, k] * A[k, j]
    return A


def dense_ic0(A):
    """IC(0) of a dense symmetric matrix on the pattern of its lower triangle, in A's dtype: L overwrites the lower triangle."""
    A = np.array(A, copy=True)
    n = A.shape[0]
    S = A != 0
    for i in range(n):
        for k in range(i):
            if not S[i, k]:
                continue
            A[i, k] = A[i, k] / A[k, k]
            for j in range(k + 1, i):
                if S[i, j] and S[j, k]:
                    A[i, j] = A[i, j] - A[i, k] * A[j, k]
            A[i, i] = A[i, i] - A[i, k] * A[i, k]
        A[i, i] = np.sqrt(A[i, i])
    return A


# ---------------------------------------------------------------------------------------------------- test matrices
def dominant(off, col, dtype, seed, base=0):
    """Values on the pattern: off-diagonals in [-1, 0), the diagonal 1 + the row's absolute sum (and the column's, so that the
    matrix stays dominant when only the lower triangle is read)."""
    offz, colz, n, rowof = _pattern(off, col, base)
    rng = np.random.default_rng(seed)
    v = -rng.random(colz.size)
    s = np.bincount(rowof, weights=np.abs(v), minlength=n) + np.bincount(colz, weights=np.abs(v), minlength=n)
    dg = colz == rowof
    v[dg] = 1.0 + s[rowof[dg]]
    return v.astype(dtype)


def chain(n, base=0):
    """Lower bidiagonal: row 0 stores (0, 0), row i > 0 stores (i, i - 1) and (i, i); n levels."""
    i = np.arange(1, n)
    off = np.concatenate([[0], 1 + 2 * np.arange(n)]).astype(np.int32)
    col = np.concatenate([[0], np.stack([i - 1, i], axis=1).ravel()]).astype(np.int32)
    return off + base, col + base


def diagonal(n, base=0):
    return (np.arange(n + 1, dtype=np.int32) + base), (np.arange(n, dtype=np.int32) + base)


def with_diagonal(off, col, n):
    """The CSR pattern with every missing diagonal added, columns sorted."""
    off = np.asarray(off, np.int64)
    col = np.asarray(col, np.int64)
    rowof = np.repeat(np.arange(n), np.diff(off))
    r = np.concatenate([rowof, np.arange(n)])
    c = np.concatenate([col, np.arange(n)])
    key = np.unique(r * n + c)
    r, c = key // n, key % n
    o = np.concatenate([[0], np.cumsum(np.bincount(r, minlength=n))])
    return o.astype(np.int32), c.astype(np.int32)
