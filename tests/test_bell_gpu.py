"""GPU: the native Blocked-ELL SpMM of libb200spmv.so (b200spmm_bell, cusparseSpMM on a Blocked-ELL matA) bit for bit against the
int64 reference of oracle/bell_ref.py over every type combination, block size, pipeline and tile edge, layout, base, scalar mode and
misaligned view; NaN where nothing may be read; against the closed library within the fp32 accumulation bound; status parity;
repeatability and graph replay; forwarded kinds; the reference sample."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest
import torch

from cudalibrarysamples_b200 import cusparse_api as cs
from cudalibrarysamples_b200 import lib as _lib
from oracle import bell_ref as R

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEV = torch.device("cuda:0")
ROW, COL = cs.CUSPARSE_ORDER_ROW, cs.CUSPARSE_ORDER_COL
NT, TR = cs.CUSPARSE_OPERATION_NON_TRANSPOSE, cs.CUSPARSE_OPERATION_TRANSPOSE
# (A / B type, C type, output kind of the exactness check)
TYPES = {"f16-f16": (torch.float16, torch.float16, "f16"), "f16-f32": (torch.float16, torch.float32, "f32"),
         "bf16-bf16": (torch.bfloat16, torch.bfloat16, "bf16"), "bf16-f32": (torch.bfloat16, torch.float32, "f32")}
CODE = {torch.float16: cs.CUDA_R_16F, torch.bfloat16: cs.CUDA_R_16BF, torch.float32: cs.CUDA_R_32F}
SCALAR_BS = [1, 2, 4, 8]
TENSOR_BS = [16, 32, 64, 128]


def P():
    return R.params()


def dense_buf(M, order, dt, pad=0, shift=0, fill=float("nan"), align=1):
    """(1-D view `shift` elements into its allocation, ld) holding the 2-D float array M (NaN allowed) in `order`, ld the tight one
    plus `pad` rounded up to a multiple of `align`; every unused slot (ld padding, the shifted head, one tail element) holds `fill`"""
    r, c = M.shape
    ld = -(-max((c if order == ROW else r) + pad, 1) // align) * align
    size = (r if order == ROW else c) * ld
    buf = torch.full((shift + size + 1,), fill, dtype=torch.float32)
    body = buf[shift:shift + size].view(-1, ld)
    body[:, :c if order == ROW else r] = torch.tensor(M if order == ROW else M.T, dtype=torch.float32)
    t = buf.to(dt).to(DEV)
    return t[shift:], ld


def read_c(t, rows, n, order, ld):
    x = t.float().cpu().numpy()
    if order == ROW:
        return x[:rows * ld].reshape(rows, ld)[:, :n]
    return x[:n * ld].reshape(n, ld)[:, :rows].T


def layer2(at, ct, rows, cols, n, bs, ell_cols, ci, vals, base, alpha, beta, B, ldb, ob, Cb, ldc, oc):
    lib = _lib.shim()
    dev = isinstance(alpha, torch.Tensor)
    ka, kb = (None, None) if dev else (C.c_float(alpha), C.c_float(beta))
    pa = alpha.data_ptr() if dev else C.addressof(ka)
    pb = beta.data_ptr() if dev else C.addressof(kb)
    rc = lib.b200spmm_bell(torch.cuda.current_stream().cuda_stream, CODE[at], CODE[ct], rows, cols, n, bs, ell_cols, ci.data_ptr(),
                           vals.data_ptr(), base, pa, pb, int(dev), B.data_ptr(), ldb, int(ob == ROW), Cb.data_ptr(), ldc, int(oc == ROW))
    torch.cuda.synchronize()
    return rc


def make(types, nbr, nbc, eb, live, bs, n, seed, base=0, lo=-1, hi=1):
    """integer inputs of a case; NaN in every value the product must not read"""
    at, ct, kind = TYPES[types]
    rows, cols = nbr * bs, nbc * bs
    ci = R.structure(nbr, nbc, eb, live, seed, base)
    a, b, c0 = R.values(rows, eb * bs, cols, n, seed + 1, lo, hi)
    af = a.astype(np.float64)
    for br in range(nbr):                                    # padding slots hold NaN
        for j in range(eb):
            if ci[br, j] == -1:
                af[br * bs:(br + 1) * bs, j * bs:(j + 1) * bs] = np.nan
    bf = b.astype(np.float64)
    used = np.zeros(nbc, bool)
    used[ci[ci != -1] - base] = True
    for c in np.flatnonzero(~used):                          # B rows no block references hold NaN
        bf[c * bs:(c + 1) * bs] = np.nan
    return dict(at=at, ct=ct, kind=kind, rows=rows, cols=cols, n=n, bs=bs, eb=eb, ci=ci, a=a, b=b, c0=c0, af=af, bf=bf, base=base)


def run(case, alpha=1.0, beta=0.0, ob=COL, oc=COL, pad=0, shift=0, device_scalars=False, via=("layer2", "shim"), align=1):
    """the case through b200spmm_bell and, where the route keeps it native, through cusparseSpMM; bit equality with the int64
    reference, and C's padding untouched.  Device scalars run through b200spmm_bell only: the closed library's
    cusparseSpMM_bufferSize refuses device pointer mode for a Blocked-ELL A (NOT_SUPPORTED), so no sample can reach it."""
    c = case
    if device_scalars:
        via = tuple(v for v in via if v != "shim")
    rows, cols, n, bs, eb, base = c["rows"], c["cols"], c["n"], c["bs"], c["eb"], c["base"]
    R.check_exact(rows, cols, bs, c["ci"] + 0, c["a"], c["b"], c["c0"], alpha, beta, c["kind"], base)
    ref = R.reference(rows, cols, bs, c["ci"], c["a"], c["b"], c["c0"], alpha, beta, base)
    ci = torch.tensor(c["ci"].ravel(), dtype=torch.int32, device=DEV)
    vals = torch.tensor(c["af"].ravel(), dtype=torch.float32).to(c["at"]).to(DEV)
    if shift:
        vals = torch.cat([torch.full((shift,), float("nan"), dtype=c["at"], device=DEV), vals])[shift:]
    B, ldb = dense_buf(c["bf"], ob, c["at"], pad, shift, align=align)
    al, be = alpha, beta
    if device_scalars:
        al, be = torch.tensor([alpha], device=DEV), torch.tensor([beta], device=DEV)
    for v in via:
        c0 = np.full((rows, n), np.nan) if beta == 0 else c["c0"].astype(np.float64)
        Cb, ldc = dense_buf(c0, oc, c["ct"], pad, 0, fill=-7.0, align=align)
        if v == "layer2":
            assert layer2(c["at"], c["ct"], rows, cols, n, bs, eb * bs, ci, vals, base, al, be, B, ldb, ob, Cb, ldc, oc) == 0
        else:
            api = cs.Api("b200")
            api.reset_stats()
            native = bell_route_native(api, c, B, ldb, ob, Cb, ldc, oc, vals, ci)
            cs.spmm_bell(api, rows, cols, bs, eb * bs, ci, vals, B, Cb, n, alpha=al, beta=be, order_b=ob, order_c=oc, ldb=ldb, ldc=ldc,
                         base=base)
            st = api.stats()
            assert st == dict(native=int(native), forwarded=int(not native), analyze=0), st
            if not native:
                continue
        got = read_c(Cb, rows, n, oc, ldc)
        assert np.array_equal(got, ref), (v, np.argwhere(got != ref)[:8])
        whole = Cb.float().cpu().numpy()
        inner = read_c(Cb, rows, n, oc, ldc)
        assert np.isfinite(inner).all()
        if ldc > (n if oc == ROW else rows):                 # ld padding of C keeps its fill
            x = whole[:(rows if oc == ROW else n) * ldc].reshape(-1, ldc)[:, (n if oc == ROW else rows):]
            assert (x == -7.0).all()


def bell_route_native(api, c, B, ldb, ob, Cb, ldc, oc, vals, ci):
    """b200spmm_bell_route for the descriptors spmm_bell creates"""
    h = api.cusparseCreate()
    matA = api.cusparseCreateBlockedEll(c["rows"], c["cols"], c["bs"], c["eb"] * c["bs"], ci, vals, c["base"])
    matB = api.cusparseCreateDnMat(c["cols"], c["n"], ldb, B, ob)
    matC = api.cusparseCreateDnMat(c["rows"], c["n"], ldc, Cb, oc)
    r = _lib.shim().b200spmm_bell_route(matA, matB, matC, NT, NT, cs.CUDA_R_32F, 0)
    api.cusparseDestroySpMat(matA)
    api.cusparseDestroyDnMat(matB)
    api.cusparseDestroyDnMat(matC)
    api.cusparseDestroy(h)
    return r == 1


# ---------------------------------------------------------------------------------------------- exact sweeps
@pytest.mark.parametrize("types", list(TYPES))
@pytest.mark.parametrize("bs", SCALAR_BS + TENSOR_BS)
def test_types_and_block_sizes_exact(types, bs):
    """every type combination and block size, -1 first / middle / last and an all-empty block-row, each B / C order, N 1, 7, 8"""
    nbr = 5 if bs <= 32 else 3
    case = make(types, nbr, 6, 4, [2, 0, 3, 4, 1], bs, 8, seed=bs)
    for ob, oc, n in ((COL, COL, 8), (ROW, ROW, 7), (ROW, COL, 1), (COL, ROW, 8)):
        c = dict(case, n=n, b=case["b"][:, :n], bf=case["bf"][:, :n], c0=case["c0"][:, :n])
        run(c, alpha=-1.0, beta=1.0, ob=ob, oc=oc)


@pytest.mark.parametrize("types", ["f16-f16", "bf16-f32"])
@pytest.mark.parametrize("bs", [16, 64])
@pytest.mark.parametrize("order", [COL, ROW], ids=["col", "row"])
def test_n_tile_edges_exact(types, bs, order):
    t = P()["n_tile"]
    for n in (1, 7, 8, t - 1, t, t + 1, 3 * t + 5):
        run(make(types, 2, 4, 3, [3, 1], bs, n, seed=n), ob=order, oc=order)


@pytest.mark.parametrize("bs", [16, 32])
def test_pipeline_depth_edges_exact(bs):
    """stored blocks per block-row around the pipeline depth: slabs = blocks * bs / 16"""
    s = P()["stages"]
    counts = sorted({0, 1, s - 2, s - 1, s, s + 1, 3 * s + 1} - {-1})
    eb = max(counts) + 2
    run(make("f16-f32", len(counts), eb + 3, eb, counts, bs, 24, seed=3), alpha=2.0, beta=0.5)


def test_block_row_counts_exact():
    """rows-per-CTA edges: block-row counts 1, 2, 3, 9 at bs 16 .. 128 (a CTA owns min(bs, max_rows_per_cta) rows)"""
    for bs in TENSOR_BS:
        for nbr in (1, 2, 3, 9):
            run(make("bf16-bf16", nbr, 3, 2, [2, 1, 0], bs, 9, seed=nbr + bs), via=("layer2",))


@pytest.mark.parametrize("ob", [COL, ROW], ids=["Bcol", "Brow"])
@pytest.mark.parametrize("oc", [COL, ROW], ids=["Ccol", "Crow"])
@pytest.mark.parametrize("base", [0, 1])
@pytest.mark.parametrize("device_scalars", [False, True], ids=["host", "device"])
def test_layouts_base_and_scalars_exact(ob, oc, base, device_scalars):
    """padded ld rounded up to a multiple of 8, so bs = 32 runs on the tensor path: base 1, device scalars, padded ldb / ldc, and at
    N = 19 a row-major B whose last 16-byte chunk is partial (3 of 8 columns)"""
    for bs in (4, 32):
        case = make("f16-f16", 4, 5, 3, [3, 0, 2, 1], bs, 19, seed=5, base=base)
        for alpha, beta in R.SCALARS:
            run(case, alpha=alpha, beta=beta, ob=ob, oc=oc, pad=1, align=8, device_scalars=device_scalars)


@pytest.mark.parametrize("types", list(TYPES))
def test_misaligned_views_take_the_scalar_path_exact(types):
    """values and B one element into their allocation (no 16-byte cp.async possible), and an odd ldb: same bits"""
    case = make(types, 3, 4, 3, [2, 3, 0], 32, 20, seed=9)
    run(case, shift=1, ob=ROW, oc=COL)
    run(case, shift=1, ob=COL, oc=ROW, alpha=2.0, beta=0.5)
    run(case, pad=1, ob=ROW, oc=ROW)


def test_reference_sample_through_the_shim():
    E = R.samples()["spmm_blockedell"]
    api = cs.Api("b200")
    api.reset_stats()
    c = cs.spmm_bell(api, E["rows"], E["cols"], E["bs"], E["ell_cols"], torch.tensor(E["col_ind"], dtype=torch.int32, device=DEV),
                     torch.tensor(E["values"], dtype=torch.float16, device=DEV), torch.tensor(E["B_colmajor"], dtype=torch.float16, device=DEV),
                     torch.zeros(12, dtype=torch.float16, device=DEV), E["n"])
    assert np.array_equal(c.float().cpu().numpy(), E["C_result_colmajor"])
    assert api.stats()["forwarded"] == 0


# ---------------------------------------------------------------------------------------------- the closed library
MANT = {torch.float16: (10, -14), torch.bfloat16: (7, -126), torch.float32: (23, -126)}     # mantissa bits, smallest normal exponent


def ulp(x, ct):
    """one unit in the last place of C's type at magnitude x (subnormal spacing below the normal range)"""
    m, emin = MANT[ct]
    e = np.floor(np.log2(np.maximum(x, 2.0 ** emin)))
    return 2.0 ** (np.maximum(e, emin) - m)


def random_case(types, rows, bs, n, order, ci, seed):
    """random non-integer A values and B in [-1, 1), stored in A / B's type; the fp64 product and its tolerance: the fp32
    accumulation bound k * 2^-24 * |A| @ |B| plus one ulp of C's type"""
    at, ct, _ = TYPES[types]
    eb = ci.shape[1]
    rng = np.random.default_rng(seed)
    a = torch.tensor(rng.uniform(-1, 1, (rows, eb * bs)), dtype=torch.float32).to(at)
    b = torch.tensor(rng.uniform(-1, 1, (rows, n)), dtype=torch.float32).to(at)
    af, bf = a.double().numpy(), b.double().numpy()
    dense = R.to_dense(rows, rows, bs, ci, af, dtype=np.float64)
    ref = dense @ bf
    k = max(int((ci != -1).sum(axis=1).max()) * bs, 1)
    bound = k * 2.0 ** -24 * (np.abs(dense) @ np.abs(bf))
    B, ldb = dense_buf(bf, order, at)
    return dict(vals=a.to(DEV), ci=torch.tensor(ci.ravel(), dtype=torch.int32, device=DEV), B=B, ldb=ldb, ref=ref,
                tol=bound + ulp(np.abs(ref) + bound, ct))


def ours_layer2(types, rows, bs, n, order, rc):
    at, ct, _ = TYPES[types]
    Cb, ldc = dense_buf(np.zeros((rows, n)), order, ct)
    assert layer2(at, ct, rows, rows, n, bs, rc["vals"].numel() // rows, rc["ci"], rc["vals"], 0, 1.0, 0.0, rc["B"], rc["ldb"], order,
                  Cb, ldc, order) == 0
    return read_c(Cb, rows, n, order, ldc).astype(np.float64)


def closed(types, rows, bs, n, order, rc, api=None):
    at, ct, _ = TYPES[types]
    Cb, ldc = dense_buf(np.zeros((rows, n)), order, ct)
    cs.spmm_bell(api or cs.Api("cusparse"), rows, rows, bs, rc["vals"].numel() // rows, rc["ci"], rc["vals"], rc["B"], Cb, n,
                 order_b=order, order_c=order, ldb=rc["ldb"], ldc=ldc)
    return read_c(Cb, rows, n, order, ldc).astype(np.float64)


def within(got, rc, who):
    err = np.abs(got - rc["ref"])
    assert (err <= rc["tol"]).all(), (who, err.max(), (err / rc["tol"]).max())


@pytest.mark.parametrize("types", list(TYPES))
@pytest.mark.parametrize("bs", [2, 16, 32, 64])
@pytest.mark.parametrize("order", [COL, ROW], ids=["col", "row"])
def test_parity_with_the_closed_library(types, bs, order):
    """512 x 512 on random data, a shape the route forwards: ours through b200spmm_bell (scalar path at bs 2, tensor path above),
    the closed library through cusparseSpMM, both within the fp32 accumulation bound plus one ulp of C's type against fp64"""
    rows, n = 512, 72
    nbc = rows // bs
    eb = max(1, nbc // 4)
    # every slot stored, block columns ascending: the structures on which the closed library agrees with fp64 (DESIGN.md 3.14)
    full = random_case(types, rows, bs, n, order, np.sort(R.structure(nbc, nbc, eb, [eb], 11), axis=1), 12)
    within(ours_layer2(types, rows, bs, n, order, full), full, "b200")
    within(closed(types, rows, bs, n, order, full), full, "cusparse")
    # ours also with -1 slots anywhere and all-empty block-rows
    holes = random_case(types, rows, bs, n, order, R.structure(nbc, nbc, eb + 2, [eb, 1, 0, eb // 2], 13), 14)
    within(ours_layer2(types, rows, bs, n, order, holes), holes, "b200")


@pytest.mark.parametrize("types", list(TYPES))
@pytest.mark.parametrize("bs,order,n", [(2, COL, 72), (2, ROW, 8), (16, COL, 72), (16, ROW, 72)],
                         ids=["bs2-col", "bs2-row-n8", "bs16-col", "bs16-row"])
def test_parity_at_a_natively_routed_shape(types, bs, order, n):
    """64 x 64 in each class the route keeps native: cusparseSpMM through the shim runs b200spmm_bell (native 1, forwarded 0)"""
    rows = 64
    nbc = rows // bs
    eb = max(1, nbc // 2)
    rc = random_case(types, rows, bs, n, order, np.sort(R.structure(nbc, nbc, eb, [eb], 15), axis=1), 16)
    api = cs.Api("b200")
    api.reset_stats()
    got = closed(types, rows, bs, n, order, rc, api=api)
    assert api.stats() == dict(native=1, forwarded=0, analyze=0), api.stats()
    within(got, rc, "b200 via cusparseSpMM")
    within(closed(types, rows, bs, n, order, rc), rc, "cusparse")


def test_status_parity_for_shape_mismatches():
    """each mismatch: the same status from both libraries at bufferSize and at the call"""
    ci = torch.tensor([1, 0], dtype=torch.int32, device=DEV)
    v = torch.ones(8, dtype=torch.float16, device=DEV)
    X_ = torch.zeros(4096, dtype=torch.float16, device=DEV)
    buf = torch.zeros(1 << 20, dtype=torch.uint8, device=DEV)
    cases = {"ok": (4, 3, 4, 3), "b_rows": (6, 3, 4, 3), "c_rows": (4, 3, 6, 3), "n_mismatch": (4, 3, 4, 5)}
    for name, (br, bc, cr, cc) in cases.items():
        out = {}
        for impl in ("b200", "cusparse"):
            api = cs.Api(impl)
            h = api.cusparseCreate()
            matA = api.cusparseCreateBlockedEll(4, 4, 2, 2, ci, v)
            matB = api.cusparseCreateDnMat(br, bc, br, X_, COL)
            matC = api.cusparseCreateDnMat(cr, cc, cr, X_, COL)
            one, zero = C.c_float(1.0), C.c_float(0.0)
            st = [api.lib.cusparseSpMM_bufferSize(h, NT, NT, C.byref(one), matA, matB, C.byref(zero), matC, cs.CUDA_R_32F, 0,
                                                  C.byref(C.c_size_t(0))),
                  api.lib.cusparseSpMM(h, NT, NT, C.byref(one), matA, matB, C.byref(zero), matC, cs.CUDA_R_32F, 0,
                                       C.c_void_p(buf.data_ptr()))]
            torch.cuda.synchronize()
            api.cusparseDestroySpMat(matA)
            api.cusparseDestroyDnMat(matB)
            api.cusparseDestroyDnMat(matC)
            api.cusparseDestroy(h)
            out[impl] = st
        assert out["b200"] == out["cusparse"], (name, out)


# ---------------------------------------------------------------------------------------------- repeatability and graphs
@pytest.mark.parametrize("bs", [4, 64])
def test_repeated_calls_and_graph_replay_give_identical_bits(bs):
    rows = cols = 4096
    n = 96
    nbr, nbc = rows // bs, cols // bs
    eb = max(2, nbc // 8)
    ci = torch.tensor(R.structure(nbr, nbc, eb, [eb, eb // 2, 1], 21).ravel(), dtype=torch.int32, device=DEV)
    g = torch.Generator(device=DEV).manual_seed(22)
    vals = (torch.rand(rows * eb * bs, device=DEV, generator=g) - 0.5).half()
    B = (torch.rand(cols * n, device=DEV, generator=g) - 0.5).half()
    Cb = torch.zeros(rows * n, dtype=torch.float16, device=DEV)
    lib = _lib.shim()
    al, be = C.c_float(1.5), C.c_float(0.0)

    def call():
        return lib.b200spmm_bell(torch.cuda.current_stream().cuda_stream, cs.CUDA_R_16F, cs.CUDA_R_16F, rows, cols, n, bs, eb * bs,
                                 ci.data_ptr(), vals.data_ptr(), 0, C.addressof(al), C.addressof(be), 0, B.data_ptr(), cols, 0,
                                 Cb.data_ptr(), rows, 0)
    assert call() == 0
    torch.cuda.synchronize()
    first = Cb.clone()
    for _ in range(3):
        assert call() == 0
    torch.cuda.synchronize()
    assert torch.equal(Cb, first)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    gr = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s):
        with torch.cuda.graph(gr, stream=s):
            assert call() == 0
    Cb.fill_(float("nan"))
    for _ in range(3):
        gr.replay()
    torch.cuda.synchronize()
    assert torch.equal(Cb, first)


# ---------------------------------------------------------------------------------------------- forwarded kinds
def test_forwarded_kinds_are_counted():
    ci = torch.tensor([1, 0], dtype=torch.int32, device=DEV)
    api = cs.Api("b200")

    def once(vt=torch.float16, ct=torch.float16, compute=cs.CUDA_R_32F, opA=NT, opB=NT, alg=0, batch=1, ci=ci):
        h = api.cusparseCreate()
        v = torch.ones(8, dtype=vt, device=DEV)
        Bx = torch.ones(4096, dtype=vt, device=DEV)
        Cx = torch.zeros(4096, dtype=ct, device=DEV)
        matA = api.cusparseCreateBlockedEll(4, 4, 2, 2, ci, v)
        matB = api.cusparseCreateDnMat(4, 4, 4, Bx, COL)
        matC = api.cusparseCreateDnMat(4, 4, 4, Cx, COL)
        if batch > 1:
            api.cusparseDnMatSetStridedBatch(matB, batch, 16)
            api.cusparseDnMatSetStridedBatch(matC, batch, 16)
        api.reset_stats()
        one, zero = C.c_float(1.0), C.c_float(0.0)
        if compute == cs.CUDA_R_16F:
            one, zero = C.c_uint16(0x3C00), C.c_uint16(0)
        buf = torch.zeros(1 << 20, dtype=torch.uint8, device=DEV)
        api.lib.cusparseSpMM(h, opA, opB, C.byref(one), matA, matB, C.byref(zero), matC, compute, alg, C.c_void_p(buf.data_ptr()))
        torch.cuda.synchronize()
        st = api.stats()
        api.cusparseDestroySpMat(matA)
        api.cusparseDestroyDnMat(matB)
        api.cusparseDestroyDnMat(matC)
        api.cusparseDestroy(h)
        return st

    assert once() == dict(native=1, forwarded=0, analyze=0)
    assert once(alg=cs.CUSPARSE_SPMM_BLOCKED_ELL_ALG1) == dict(native=1, forwarded=0, analyze=0)
    assert once(ct=torch.float32) == dict(native=1, forwarded=0, analyze=0)
    assert once(compute=cs.CUDA_R_16F)["forwarded"] == 1                    # 16-bit compute
    assert once(vt=torch.float32, ct=torch.float32)["forwarded"] == 1       # fp32 Blocked-ELL
    assert once(opB=TR)["forwarded"] == 1                                   # transposed B
    assert once(opA=TR)["forwarded"] == 1
    assert once(alg=cs.CUSPARSE_SPMM_CSR_ALG2)["forwarded"] == 1           # another algorithm
    assert once(batch=2)["forwarded"] == 1                                  # strided batches


# ---------------------------------------------------------------------------------------------- the reference sample
def test_reference_sample_runs_natively():
    out = {}
    for lib in ("cusparse", "b200"):
        exe = os.path.join(ROOT, "oracle", "_ref", f"spmm_blockedell_example.{lib}")
        if not os.path.exists(exe):
            pytest.skip("oracle/_ref not built")
        env = {k: v for k, v in os.environ.items() if not k.startswith("B200SPMV_")}
        env["B200SPMV_LOG"] = "1"
        p = subprocess.run([exe], capture_output=True, text=True, timeout=120, env=env)
        assert p.returncode == 0, p.stdout + p.stderr
        assert "spmm_blockedell_example test PASSED" in p.stdout
        out[lib] = p.stderr
    assert "[b200spmv] SpMM Blocked-ELL b200spmm_bell" in out["b200"] and "forwarded" not in out["b200"], out["b200"]
