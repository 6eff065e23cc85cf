"""oracle/limits.py -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

Inputs and an exact reference for running the sparse routes at the edges of their 32-bit index and launch ranges
(tests/test_limits_gpu.py), where the arrays are gigabytes long.  Everything is a closed-form function of the entry index, built
with torch on whichever device the index tensor lives on, so nothing of that size crosses PCIe and the CPU test
(tests/test_limits_cpu.py) runs the same formulas at small sizes against scipy.

Exactness: |val| <= 3, |x| <= 3, alpha = -2, beta = 3, every row at most 2048 entries long and every column at most
~34K entries deep (fan-in, for A^T).  Every partial sum then stays below 2^24, so fp32, fp64 and every summation order (atomics
included) give the same integer, and a kernel is compared with the int64 reference bit for bit.  No value is zero, so a dropped or
duplicated product always shows.
"""
from __future__ import annotations

import math

import torch

INT32_MAX = 2**31 - 1
ALPHA, BETA = -2, 3
CHUNK = 1 << 26                      # entries per step of the generators and the reference
HOT = 4096                           # columns 0 .. HOT-1 get one entry in 16 on top of the spread (a hot set for the flat kernel)
_P = 2654435761                      # odd: k -> k * _P mod 2^j is a permutation of every 2^j consecutive k


def small(i: torch.Tensor) -> torch.Tensor:
    """1, 2, 3, -1, -2, -3 by i mod 6 (int64): the values of A, x and y0, never zero"""
    t = i % 6
    return torch.where(t < 3, t + 1, 2 - t)


def val_at(k: torch.Tensor) -> torch.Tensor:
    return small(k)


def x_at(j: torch.Tensor) -> torch.Tensor:
    return small(5 * j + 1)


def y0_at(i: torch.Tensor) -> torch.Tensor:
    return small(i + 2)


def col_at(k: torch.Tensor, cols: int) -> torch.Tensor:
    """column (base 0) of entry k: one entry in 16 on the hot columns 0 .. HOT-1, the rest spread by a multiplicative hash; entries
    1, 2 and 3 sit on cols - 1, 2^31 - 1 and 2^31 where those columns exist, entry 0 on column 0"""
    hot = min(HOT, cols)
    c = torch.where(k % 16 == 0, (k // 16) % hot, (k * _P) % cols)
    c = torch.where(k == 1, torch.full_like(k, cols - 1), c)
    if cols > 2**31 - 1:
        c = torch.where(k == 2, torch.full_like(k, 2**31 - 1), c)
    if cols > 2**31:
        c = torch.where(k == 3, torch.full_like(k, 2**31), c)
    return c


def fill(out: torch.Tensor, fn, start: int = 0) -> torch.Tensor:
    """out[i] = fn(start + i) (int64 index) in chunks of CHUNK entries"""
    n = out.numel()
    for s in range(0, n, CHUNK):
        e = min(n, s + CHUNK)
        k = torch.arange(start + s, start + e, dtype=torch.int64, device=out.device)
        out[s:e] = fn(k).to(out.dtype)
    return out


def offsets(kind: str, rows: int, nnz: int, device="cpu") -> torch.Tensor:
    """int64 row offsets (base 0, rows + 1 entries, off[rows] = nnz) of a profile:
      uniform  : floor(i * nnz / rows), row rows // 2 emptied (its entries go to the next row);
      skewed   : row lengths growing linearly from ~nnz / (9 rows) to ~2 nnz / rows (a quadratic off), row rows // 2 emptied;
      ends     : 16 entries in each of the first and the last 10 rows, every other row empty (nnz = 320)."""
    i = torch.arange(rows + 1, dtype=torch.int64, device=device)
    if kind == "uniform":
        off = i * nnz // rows
    elif kind == "skewed":
        c = rows // 8
        off = torch.floor((i * (i + c)).double() / (float(rows) * float(rows + c)) * nnz).long()
        off[-1] = nnz
    elif kind == "ends":
        assert nnz == 320 and rows >= 20
        return 16 * torch.clamp(i, max=10) + 16 * torch.clamp(i - (rows - 10), min=0)
    else:
        raise ValueError(kind)
    e = rows // 2
    off[e + 1] = off[e]
    return off


def max_row(off: torch.Tensor) -> int:
    return int((off[1:] - off[:-1]).max())


def reference(off: torch.Tensor, col: torch.Tensor, val: torch.Tensor, x: torch.Tensor, n_out: int, transpose: bool = False,
              base: int = 0, y0: torch.Tensor | None = None, alpha: int = ALPHA, beta: int = BETA) -> torch.Tensor:
    """int64 alpha * op(A) x + beta * y0 of a CSR matrix (off base 0, int64; col / val / x of any type holding integers, col with
    `base`), n_out = rows (op N) or cols (op T); y0 None: beta = 0.  Chunked: the row of each entry from searchsorted on the
    offsets, the products summed with index_add_."""
    acc = torch.zeros(n_out, dtype=torch.int64, device=off.device)
    nnz = int(off[-1])
    for s in range(0, nnz, CHUNK):
        e = min(nnz, s + CHUNK)
        k = torch.arange(s, e, dtype=torch.int64, device=off.device)
        r = torch.searchsorted(off, k, right=True) - 1
        c = col[s:e].long() - base
        if transpose:
            acc.index_add_(0, c, val[s:e].long() * x[r].long())
        else:
            acc.index_add_(0, r, val[s:e].long() * x[c].long())
    y = alpha * acc
    return y if y0 is None else y + beta * y0.long()


def reference_entries(n_entries: int, row_col, val: torch.Tensor, x: torch.Tensor, n_out: int, transpose: bool = False,
                      device="cuda") -> torch.Tensor:
    """int64 alpha * op(A) x (beta = 0) of an entry list: row_col(k) gives the (row, column) of entries k (int64, base 0; a column
    < 0 marks a padding slot, skipped), val[k] their values.  Chunked like `reference`."""
    acc = torch.zeros(n_out, dtype=torch.int64, device=device)
    for s in range(0, n_entries, CHUNK):
        e = min(n_entries, s + CHUNK)
        k = torch.arange(s, e, dtype=torch.int64, device=device)
        r, c = row_col(k)
        live = c >= 0
        r, c, v = r[live], c[live], val[s:e].long()[live]
        if transpose:
            acc.index_add_(0, c, v * x[r].long())
        else:
            acc.index_add_(0, r, v * x[c].long())
    return ALPHA * acc


def sell_row_col(col: torch.Tensor, slice_size: int, width: int):
    """row_col of a Sliced-ELL layout with every slice `width` wide: entry i = slice s, column slot j, row s * S + i mod S"""
    per = slice_size * width

    def rc(k):
        return (k // per) * slice_size + (k % per) % slice_size, col[int(k[0]):int(k[-1]) + 1].long()
    return rc


def bound_ok(off: torch.Tensor, col_fan_in: int | None = None) -> bool:
    """the exactness precondition: 9 * |alpha| * (longest row, or deepest column for A^T) + 3 * |beta| < 2^24"""
    longest = max(max_row(off), col_fan_in or 0)
    return 9 * abs(ALPHA) * longest + 3 * abs(BETA) < 2**24


def gb(nbytes: float) -> float:
    return nbytes / 1e9


def round_up_256(b: int) -> int:
    return (b + 255) // 256 * 256


def spread_fan_in(nnz: int, cols: int) -> int:
    """an upper bound of the entries col_at puts on one column among the first nnz (for the A^T bound)"""
    hot = min(HOT, cols)
    return math.ceil(nnz / cols) + 1 + math.ceil(nnz / 16 / hot) + 1 + 3
