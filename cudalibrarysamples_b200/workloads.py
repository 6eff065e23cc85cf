"""Synthetic workloads of BASELINE.json's configs, generated ON the GPU (b200gen_* kernels + torch for sort/scan).

Bit-identical to the CPU generators of the checker (oracle/oracle.py) -- tests/test_parity_gpu.py compares them -- so the
full-size matrices never cross PCIe.  torch is plumbing here (memory, sort, cumsum), not the product.

  config 2 / target : R-MAT, (a,b,c,d)=(0.57,0.19,0.19,0.05), rows x rows, avg 16 nnz/row, fp64  (SURVEY.md 8d)
  config 3          : 7-pt Laplacian nx^3 (cuDSS/simple_residual/laplace_generator.hxx:34-107) -> Sliced-ELL, slice 32
  config 4          : 5-pt Laplacian grid^2 (cuSPARSE/cg/cg_example.c:71-128)
"""
from __future__ import annotations

import math

import torch

from . import lib as _lib

RMAT_ABCD = (0.57, 0.19, 0.19, 0.05)
RMAT_OVERSAMPLE = 1.5


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _check(rc, what):
    if rc != 0:
        raise RuntimeError(f"{what} failed with code {rc}")


def _dt(dtype):
    return {torch.float32: 0, torch.float64: 1}[dtype]


def rmat_thresholds(abcd=RMAT_ABCD):
    a, b, c, _ = abcd
    two32 = 4294967296.0
    return int(a * two32), int((a + b) * two32), int((a + b + c) * two32)


def rmat_scale(n):
    return max(1, int(n - 1).bit_length())


def uniform(seed, count, dtype=torch.float64, device="cuda", i0=0):
    out = torch.empty(count, dtype=dtype, device=device)
    _check(_lib.gen().b200gen_uniform(_stream(), _dt(dtype), seed, i0, count, out.data_ptr()), "b200gen_uniform")
    return out


def rmat_csr(rows, cols=None, avg_nnz=16, seed=42, val_seed=43, dtype=torch.float64, device="cuda", abcd=RMAT_ABCD,
             chunk=1 << 26):
    """Same definition as oracle.rmat_csr: first rows*avg_nnz distinct in-range edges of the hash stream, CSR-sorted."""
    cols = rows if cols is None else cols
    scale = rmat_scale(max(rows, cols))
    target = int(rows) * int(avg_nnz)
    cand = int(math.ceil(target * RMAT_OVERSAMPLE))
    tA, tAB, tABC = rmat_thresholds(abcd)
    keys = torch.empty(cand, dtype=torch.int64, device=device)
    L = _lib.gen()
    for e0 in range(0, cand, chunk):
        n = min(chunk, cand - e0)
        _check(L.b200gen_rmat_keys(_stream(), seed, e0, n, scale, tA, tAB, tABC, rows, cols, keys.data_ptr() + 8 * e0),
               "b200gen_rmat_keys")
    # first occurrence of every valid key, in stream order
    skeys, perm = torch.sort(keys, stable=True)
    del keys
    first = torch.ones_like(skeys, dtype=torch.bool)
    first[1:] = skeys[1:] != skeys[:-1]
    first &= skeys >= 0
    first_pos = perm[first]          # stream index of each distinct key's first occurrence
    ukeys = skeys[first]
    del skeys, perm, first
    if first_pos.numel() > target:
        order = torch.argsort(first_pos)[:target]    # the `target` earliest distinct edges
        ukeys = torch.sort(ukeys[order]).values
        del order
    del first_pos
    rr = torch.div(ukeys, cols, rounding_mode="floor")
    cc = (ukeys - rr * cols).to(torch.int32)
    counts = torch.bincount(rr, minlength=rows)
    off = torch.zeros(rows + 1, dtype=torch.int64, device=device)
    off[1:] = torch.cumsum(counts, 0)
    off = off.to(torch.int32)
    val = uniform(val_seed, int(cc.numel()), dtype, device)
    return off, cc, val


def stencil5_csr(grid, mass=0.04, ux=0.0, uy=0.0, device="cuda"):
    """cg_example.c:71-128 (defaults) / bicgstab_example.c:69-127 (mass=.3, ux=.3, uy=.2); fp64 like the samples."""
    n = grid * grid
    L = _lib.gen()
    counts = torch.empty(n, dtype=torch.int32, device=device)
    _check(L.b200gen_stencil5_counts(_stream(), grid, counts.data_ptr()), "stencil5_counts")
    off = torch.zeros(n + 1, dtype=torch.int32, device=device)
    off[1:] = torch.cumsum(counts, 0, dtype=torch.int64).to(torch.int32)
    nnz = 5 * n - 4 * grid
    col = torch.empty(nnz, dtype=torch.int32, device=device)
    val = torch.empty(nnz, dtype=torch.float64, device=device)
    _check(L.b200gen_stencil5_fill(_stream(), grid, mass, ux, uy, off.data_ptr(), col.data_ptr(), val.data_ptr()),
           "stencil5_fill")
    return off, col, val


def laplace7_csr(nx, dtype=torch.float64, device="cuda"):
    """cuDSS/simple_residual/laplace_generator.hxx:34-107."""
    n = nx ** 3
    L = _lib.gen()
    counts = torch.empty(n, dtype=torch.int32, device=device)
    _check(L.b200gen_laplace7_counts(_stream(), nx, counts.data_ptr()), "laplace7_counts")
    off = torch.zeros(n + 1, dtype=torch.int32, device=device)
    off[1:] = torch.cumsum(counts, 0, dtype=torch.int64).to(torch.int32)
    nnz = int(off[-1].item())
    col = torch.empty(nnz, dtype=torch.int32, device=device)
    val = torch.empty(nnz, dtype=dtype, device=device)
    _check(L.b200gen_laplace7_fill(_stream(), _dt(dtype), nx, off.data_ptr(), col.data_ptr(), val.data_ptr()),
           "laplace7_fill")
    return off, col, val


def csr_to_coo_rows(off, base=0):
    rows = off.numel() - 1
    counts = (off[1:] - off[:-1]).to(torch.int64)
    return torch.repeat_interleave(torch.arange(rows, device=off.device, dtype=torch.int32) + base, counts)


def csr_to_sell(off, col, val, slice_size, base=0):
    """Sliced-ELL per spmv_sell_example.c:48-69 (column-major in slice, padding col=-1+base, val=0). torch plumbing."""
    dev = off.device
    rows = off.numel() - 1
    nsl = (rows + slice_size - 1) // slice_size
    o = off.to(torch.int64) - base
    lens = o[1:] - o[:-1]
    pad = nsl * slice_size - rows
    lens_p = torch.cat([lens, torch.zeros(pad, dtype=torch.int64, device=dev)]) if pad else lens
    width = lens_p.view(nsl, slice_size).max(dim=1).values
    soff = torch.zeros(nsl + 1, dtype=torch.int64, device=dev)
    soff[1:] = torch.cumsum(width * slice_size, 0)
    total = int(soff[-1].item())
    scol = torch.full((total,), -1 + base, dtype=torch.int32, device=dev)
    sval = torch.zeros(total, dtype=val.dtype, device=dev)
    nnz = col.numel()
    r = torch.repeat_interleave(torch.arange(rows, device=dev, dtype=torch.int64), lens)
    k = torch.arange(nnz, device=dev, dtype=torch.int64) - o[:-1][r]
    s = torch.div(r, slice_size, rounding_mode="floor")
    dst = soff[s] + k * slice_size + (r - s * slice_size)
    scol[dst] = col
    sval[dst] = val
    return (soff + base).to(torch.int32), scol, sval


def csr_bytes(rows, cols, nnz, vb, beta_nonzero=False, ib=4):
    """Algorithmic bytes of one CSR SpMV (SURVEY.md 8d / BASELINE.md 2.3)."""
    return nnz * (vb + ib) + (rows + 1) * ib + cols * vb + rows * vb * (2 if beta_nonzero else 1)


def sell_bytes(rows, cols, slots, nslices, vb, ib=4):
    return slots * (vb + ib) + (nslices + 1) * ib + cols * vb + rows * vb


def coo_bytes(rows, cols, nnz, vb, ib=4):
    return nnz * (vb + 2 * ib) + cols * vb + rows * vb
