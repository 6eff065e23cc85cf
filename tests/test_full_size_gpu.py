"""GPU parity at BASELINE.json's FULL sizes, through size-independent properties (the CPU oracle would need minutes
here; the small-size oracle comparisons live in test_parity_gpu.py):

  * agreement with the closed cusparseSpMV on the same device buffers (same tolerance as everywhere else),
  * linearity      A(a*x1 + b*x2) = a*A*x1 + b*A*x2,
  * row-sum check  A*1 = row sums of val (computed independently with torch.segment_reduce / index_add),
  * symmetry       <x, A*y> = <y, A*x> for the symmetric Poisson matrix of config 4.

Inputs come from the device-side generators, which test_parity_gpu.py proves bit-identical to the oracle's.
"""
import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def env():
    from cudalibrarysamples_b200 import cusparse_api as cs
    from cudalibrarysamples_b200 import workloads as W
    return cs, W, cs.Api("b200"), cs.Api("cusparse")


def rel(a, b):
    return float((torch.linalg.norm(a.double() - b.double()) / torch.linalg.norm(b.double())).item())


def spmv(cs, api, fmt, rows, cols, arrays, x, alpha=1.0, beta=0.0, y0=None):
    op = cs.SpMVOperator(api, fmt, rows, cols, arrays)
    y = torch.zeros(rows, dtype=x.dtype, device="cuda") if y0 is None else y0.clone()
    op(x, y, alpha, beta)
    torch.cuda.synchronize()
    op.close()
    return y


def test_config2_rmat_1m_fp64_csr(env):
    """BASELINE.json configs[1]: R-MAT 1,000,000 x 1,000,000, 16 M non-zeros, fp64 (the benchmark matrix)."""
    cs, W, ours, closed = env
    rows = 1_000_000
    off, col, val = W.rmat_csr(rows)
    arrays = dict(off=off, col=col, val=val)
    x1, x2 = W.uniform(44, rows), W.uniform(45, rows)
    y1 = spmv(cs, ours, "csr", rows, rows, arrays, x1)
    assert rel(y1, spmv(cs, closed, "csr", rows, rows, arrays, x1)) < 1e-12
    # linearity
    y2 = spmv(cs, ours, "csr", rows, rows, arrays, x2)
    y12 = spmv(cs, ours, "csr", rows, rows, arrays, 0.5 * x1 - 2.0 * x2)
    assert rel(y12, 0.5 * y1 - 2.0 * y2) < 1e-12
    # alpha / beta with y in place: y = -A x1 + y2  (cg_example.c:153-160)
    y3 = spmv(cs, ours, "csr", rows, rows, arrays, x1, alpha=-1.0, beta=1.0, y0=y2)
    assert rel(y3, y2 - y1) < 1e-12
    # row sums: A * 1
    ones = torch.ones(rows, dtype=torch.float64, device="cuda")
    lens = (off[1:] - off[:-1]).to(torch.int64)
    row_of = torch.repeat_interleave(torch.arange(rows, device="cuda"), lens)
    want = torch.zeros(rows, dtype=torch.float64, device="cuda").index_add_(0, row_of, val)
    assert rel(spmv(cs, ours, "csr", rows, rows, arrays, ones), want) < 1e-12
    # bit-reproducible
    assert torch.equal(y1, spmv(cs, ours, "csr", rows, rows, arrays, x1))


def test_config3_laplace7_256_fp32_sell(env):
    """BASELINE.json configs[2]: 7-pt Laplacian 256^3 (laplace_generator.hxx:34-107) as Sliced-ELL, slice 32, fp32."""
    cs, W, ours, closed = env
    nx = 256
    n = nx ** 3
    off, col, val = W.laplace7_csr(nx, torch.float32)
    so, sc, sv = W.csr_to_sell(off, col, val, 32)
    arrays = dict(off=so, col=sc, val=sv, slice_size=32, nnz=int(col.numel()))
    x = W.uniform(44, n, torch.float32)
    y = spmv(cs, ours, "sell", n, n, arrays, x)
    assert rel(y, spmv(cs, closed, "sell", n, n, arrays, x)) < 1e-5
    # the same operator in CSR must give the same vector
    assert rel(y, spmv(cs, ours, "csr", n, n, dict(off=off, col=col, val=val), x)) < 1e-5
    # interior rows of A*1 are 16 - 6 = 10 (diag 16, six -1 neighbours); every row lies in [10, 13]
    r = spmv(cs, ours, "sell", n, n, arrays, torch.ones(n, dtype=torch.float32, device="cuda"))
    assert float(r.min().item()) == 10.0 and float(r.max().item()) == 13.0


def test_config4_poisson_8192_fp64_csr(env):
    """BASELINE.json configs[3]: the operator of the CG run, 5-pt Poisson 8192^2 (cg_example.c:71-128), fp64."""
    cs, W, ours, closed = env
    g = 8192
    n = g * g
    off, col, val = W.stencil5_csr(g)
    arrays = dict(off=off, col=col, val=val)
    x, z = W.uniform(44, n), W.uniform(45, n)
    ax = spmv(cs, ours, "csr", n, n, arrays, x)
    assert rel(ax, spmv(cs, closed, "csr", n, n, arrays, x)) < 1e-12
    az = spmv(cs, ours, "csr", n, n, arrays, z)
    lhs, rhs = torch.dot(z, ax), torch.dot(x, az)          # A is symmetric
    scale = float((torch.linalg.norm(z) * torch.linalg.norm(ax)).item())
    assert abs(float((lhs - rhs).item())) <= 1e-12 * scale
    # b = 0.75 * A * 1 (cg_example.c:405-418): interior rows give 0.75 * 0.04
    b = spmv(cs, ours, "csr", n, n, arrays, torch.ones(n, dtype=torch.float64, device="cuda"), alpha=0.75)
    interior = b.view(g, g)[1:-1, 1:-1]
    assert float((interior - 0.75 * 0.04).abs().max().item()) < 1e-13


def test_config4_cg_fused_driver_matches_torch_ops(env):
    """BASELINE.json configs[3]'s CG at the size bench.py times (n = 8192^2: about 62 grid-stride passes of the fused BLAS-1
    kernels at their grid cap): 20 iterations of the fused driver (CUDA graph on) against the torch-op driver on the same
    operator, and the fused driver's recurrence norm against the true residual ||b - A x||."""
    from cudalibrarysamples_b200.cg import CgSolver, FusedCgSolver
    from cudalibrarysamples_b200.sharded import ShardedCsr
    cs, W, ours, closed = env
    g, iters = 8192, 20
    n = g * g
    off, col, val = W.stencil5_csr(g)

    def make_local(r, c, arrays):
        return cs.SpMVOperator(ours, "csr", r, c, arrays, preprocess=True)
    sh = ShardedCsr(off, col, val, 0, 1, make_local, balance="rows")
    del off, col, val
    b = sh.new_y_shard()
    sh.spmv(sh.new_x_shard(torch.ones(n, dtype=torch.float64, device="cuda")), b, alpha=0.75, beta=0.0)
    fused = FusedCgSolver(sh, b, use_graph=True)
    xf, nf = fused.run(iters)
    torch.cuda.synchronize()
    assert fused.graph_error is None, fused.graph_error
    xt, nt = CgSolver(sh, b).run(iters)
    assert abs(nf[0] - nt[0]) <= 1e-9 * nt[0] and abs(nf[-1] - nt[-1]) <= 1e-9 * nt[-1], (nf, nt[0], nt[-1])
    assert rel(xf, xt) < 1e-9
    del xt
    res = b.clone()
    sh.spmv(xf, res, alpha=-1.0, beta=1.0)                                  # b - A x
    true = float(torch.linalg.norm(res).item())
    assert true <= 1.01 * nf[-1] + 1e-12, (true, nf[-1])
    sh.close()


def test_north_star_rmat_10m_fp64_csr(env):
    """BASELINE.json north_star acceptance size: R-MAT 10,000,000 x 10,000,000, avg 16 nnz/row, fp64;
    ||y - y_ref|| / ||y_ref|| < 1e-12 against the closed library, through the preprocessed call sequence of
    spmv_csr_example.c:104-112 (the flat plan's 31-bit non-zero positions and > 2^27 non-zeros are exercised here)."""
    cs, W, ours, closed = env
    rows = 10_000_000
    off, col, val = W.rmat_csr(rows)
    assert int(col.numel()) > 150_000_000
    arrays = dict(off=off, col=col, val=val)
    x1, x2 = W.uniform(44, rows), W.uniform(45, rows)
    ours.reset_stats()
    y1 = spmv(cs, ours, "csr", rows, rows, arrays, x1)
    assert ours.stats()["forwarded"] == 0
    assert rel(y1, spmv(cs, closed, "csr", rows, rows, arrays, x1)) < 1e-12
    y2 = spmv(cs, ours, "csr", rows, rows, arrays, x2)
    y12 = spmv(cs, ours, "csr", rows, rows, arrays, 0.5 * x1 - 2.0 * x2)
    assert rel(y12, 0.5 * y1 - 2.0 * y2) < 1e-12
    # the no-preprocess path (cg_example.c style: tile plan rebuilt per call) on the same matrix
    op = cs.SpMVOperator(ours, "csr", rows, rows, arrays, preprocess=False)
    y3 = torch.zeros(rows, dtype=torch.float64, device="cuda")
    op(x1, y3, 1.0, 0.0)
    torch.cuda.synchronize()
    op.close()
    assert rel(y3, y1) < 1e-13
    assert torch.equal(y1, spmv(cs, ours, "csr", rows, rows, arrays, x1))      # bit-reproducible


def test_config5_spmm_2m_fp32_csr_times_dense(env):
    """BASELINE.json configs[4]: fp32 CSR SpMM (cuSPARSE/spmm_csr), A 2M x 2M with 32 non-zeros per row, B dense n = 64,
    column-major B and C as in spmm_csr_example.c:100-104; against the closed library on the same buffers, plus
    linearity in B and the column-by-column identity  C[:, j] = SpMV(A, B[:, j])."""
    cs, W, ours, closed = env
    rows, per_row, n = 2_000_000, 32, 64
    g = torch.Generator(device="cuda").manual_seed(5)
    col = torch.randint(0, rows, (rows, per_row), device="cuda", generator=g, dtype=torch.int32).sort(dim=1).values.reshape(-1).contiguous()
    off = (torch.arange(rows + 1, device="cuda", dtype=torch.int64) * per_row).to(torch.int32)
    val = W.uniform(43, rows * per_row, torch.float32)
    arrays = dict(off=off, col=col, val=val)
    B1, B2 = W.uniform(46, rows * n, torch.float32), W.uniform(47, rows * n, torch.float32)
    C0 = torch.zeros(rows * n, dtype=torch.float32, device="cuda")
    ours.reset_stats()
    c1 = cs.spmm(ours, rows, rows, arrays, B1, C0)
    assert ours.stats()["forwarded"] == 0
    ref = cs.spmm(closed, rows, rows, arrays, B1, C0)
    assert rel(c1, ref) < 1e-5
    del ref
    c12 = cs.spmm(ours, rows, rows, arrays, 0.5 * B1 - 2.0 * B2, C0)
    c2 = cs.spmm(ours, rows, rows, arrays, B2, C0)
    assert rel(c12, 0.5 * c1 - 2.0 * c2) < 1e-5
    del c12, c2
    for j in (0, 37, 63):                                                      # column j of C is one SpMV
        yj = spmv(cs, ours, "csr", rows, rows, arrays, B1[j * rows:(j + 1) * rows].contiguous())
        assert rel(c1[j * rows:(j + 1) * rows], yj) < 1e-5
