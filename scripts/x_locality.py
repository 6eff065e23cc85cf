#!/usr/bin/env python
"""Static locality counts of the x gather of csr_flat_kernel on the headline matrix (CPU only, no timing).

  python scripts/x_locality.py [rows] [value bytes]       default: R-MAT 1M x 1M, 16 non-zeros per row, seed 42; fp64

Prints
  - distinct 128-byte lines of x that the 8 gather instructions of a 256-non-zero warp chunk touch (summed over the 8);
  - the share of non-zeros in the hottest columns that fit 64 .. 160 KB (what the hot plan of the flat CSR kernel packs);
  - an ideal-cache model: the share of gathers that hit if a cache of 192 / 224 KB held exactly the most-used lines, for x in
    natural column order, with the hottest 128 KB of columns packed in front (the hot plan), and with every column relabelled
    by use count.  An upper bound for comparison between layouts, not a predicted hit rate."""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import oracle as O  # noqa: E402

LINE = 128


def hit_share(line_of_gather, budget_bytes):
    """share of gathers served by the budget_bytes / 128 most-used lines"""
    use = np.sort(np.bincount(line_of_gather))[::-1]
    return float(use[:budget_bytes // LINE].sum()) / line_of_gather.size


def main():
    rows = int(sys.argv[1]) if len(sys.argv) > 1 else 1_000_000
    vb = int(sys.argv[2]) if len(sys.argv) > 2 else 8
    per_line = LINE // vb
    off, col, _ = O.rmat_csr(rows, avg_nnz=16, seed=42, val_seed=43)
    nnz = col.size
    col = col.astype(np.int64)
    print(f"R-MAT {rows} x {rows}: nnz {nnz}, empty rows {int(np.count_nonzero(np.diff(off) == 0))}")

    # lines per gather instruction: 32 consecutive non-zeros, one warp instruction
    steps = nnz // 32
    lines = (col[:steps * 32] // per_line).reshape(steps, 32)
    s = np.sort(lines, axis=1)
    distinct = 1 + np.count_nonzero(np.diff(s, axis=1), axis=1)
    print(f"distinct {LINE} B lines per gather instruction: {distinct.mean():.1f} of 32 lanes; per 256-non-zero chunk: {8 * distinct.mean():.0f}")

    cnt = np.bincount(col, minlength=rows)
    order = np.argsort(-cnt, kind="stable")
    for kb in (64, 96, 128, 160):
        h = kb * 1024 // vb
        print(f"hottest {h} columns ({kb} KB): {cnt[order[:h]].sum() / nnz:.1%} of the gathers")

    h = 128 * 1024 // vb
    slot = np.full(rows, -1, np.int64)
    slot[np.sort(order[:h])] = np.arange(h)                     # the hot plan: hot columns ascending, packed in front
    packed = np.where(slot[col] >= 0, slot[col] // per_line, (col // per_line) + (h + per_line - 1) // per_line)
    rank = np.empty(rows, np.int64)
    rank[order] = np.arange(rows)
    relabelled = rank[col] // per_line
    natural = col // per_line
    for kb in (192, 224):
        b = kb * 1024
        print(f"ideal cache {kb} KB: natural order {hit_share(natural, b):.1%}, hottest {h} columns packed {hit_share(packed, b):.1%}, "
              f"all columns relabelled {hit_share(relabelled, b):.1%}")


if __name__ == "__main__":
    main()
