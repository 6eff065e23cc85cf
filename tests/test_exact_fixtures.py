"""CPU: the exact fixtures of oracle/exact.py, and the CPU emulations of the kernels held to them BIT FOR BIT.

On these inputs every partial sum is an integer the value type represents, so a correct kernel -- whatever its summation order
-- returns exactly the int64 reference.  Checked here: the exactness precondition of every fixture, that the boundary
profiles hit every boundary class they claim (recomputed from the row offsets and the constants of the built library, so a
retuned constant that moves a border shows up), and that the numpy lane emulations of csr_flat_kernel, csr_seg_kernel and
csr_short_kernel and the host-compiled source of the generic kernels reproduce the reference with np.array_equal.  The
same fixtures run on the GPU in tests/test_exact_gpu.py."""
import ctypes as C
import math

import numpy as np
import pytest

from oracle import exact as E
from oracle import oracle as O

KINDS = ["f32", "f64", "wide"]


@pytest.fixture(scope="module")
def P(built_lib):
    return E.kernel_params()


@pytest.fixture(scope="module")
def profiles(P):
    return E.boundary_profiles(P)


def edge_profiles():
    from test_parity_gpu import EDGE            # the tolerance suite's edge profiles, reused with exact values
    return {f"edge_{k}": (v, 120000) for k, v in EDGE.items()}


def all_profiles(P):
    d = dict(E.boundary_profiles(P))
    d.update(edge_profiles())
    return d


# ------------------------------------------------------------------------------------------ the fixtures themselves
def test_precondition_holds_for_every_fixture(P):
    for name, (lens, cols) in all_profiles(P).items():
        for kind in KINDS + ["mixed"]:
            f = E.Fixture(name, lens, cols, kind, seed=1)
            assert np.all(f.a != 0) and np.all(f.x != 0), (name, kind)
            assert np.all(f.y0 % 2 == 0)
            for alpha, beta in E.SCALARS:
                f.check(alpha, beta)
                if f.rows and f.cols:
                    f.check(alpha, beta, transpose=True)
            # the float views hold the integers exactly
            assert np.array_equal(f.val.astype(np.int64), f.a) and np.array_equal(f.xf().astype(np.int64), f.x)


def test_wide_fixtures_need_more_than_fp32():
    """The wide variant exists to catch an accumulator narrowed to fp32: its products and row sums must not fit 24 bits."""
    f = E.Fixture("w", np.full(50, 40), 500, "wide", seed=2)
    s = E.row_sums(f.off, f.col, f.a, f.x, absolute=True)
    assert s.min() >= 1 << 24 and np.abs(f.a).min() >= 1 << 12
    m = E.Fixture("m", np.full(50, 40), 500, "mixed", seed=2)
    assert np.abs(m.x).min() >= 1 << 30 and np.all(m.val.astype(np.int64) == m.a)
    # in fp32 the same product is not exact any more
    assert np.any(f.val.astype(np.float32)[:100] * f.xf().astype(np.float32)[f.col[:100]] != (f.a * f.x[f.col])[:100])


def test_reference_agrees_with_the_oracle(P):
    """The int64 reference is the plain product: it agrees with the C oracle (fp64) on every profile."""
    for name, (lens, cols) in E.boundary_profiles(P).items():
        f = E.Fixture(name, lens, cols, "f64", seed=1)
        for alpha, beta in E.SCALARS:
            got = f.want(alpha, beta)
            y0 = f.y0f() if beta != 0 else np.zeros(f.rows)
            assert np.array_equal(got, O.spmv_csr(f.off, f.col, f.val, f.xf(), y0, alpha, beta)), (name, alpha, beta)


def test_profiles_cover_every_boundary_class(P, profiles):
    hit = set()
    for name, (lens, cols) in profiles.items():
        off = np.concatenate([[0], np.cumsum(lens)])
        hit |= E.coverage(off, cols, P)
    missing = set(E.BOUNDARY_CLASSES) - hit
    assert not missing, f"no profile hits {sorted(missing)}"


def test_coverage_notices_a_missing_class(P, profiles):
    """The coverage check is not vacuous: without the profiles that carry them, classes go missing."""
    hit = set()
    for name, (lens, cols) in profiles.items():
        if name in ("short_block_caps", "rows_cross_borders") or name.startswith("random_mix"):
            continue
        hit |= E.coverage(np.concatenate([[0], np.cumsum(lens)]), cols, P)
    assert {"short_block_cap_m1", "short_block_2cap", "cross_cta_3+", "cross_tile_3+"} - hit


def test_emulation_constants_are_the_library_constants(P):
    """The numpy emulations restate the kernels with constants of their own: they must be the built library's."""
    import test_flat_emulation as F
    import test_seg_emulation as S
    import test_short_emulation as SH
    assert F.CHUNK == P["warp_chunk"] == P["plan_chunk"] and F.CHUNK * F.WARPS == P["cta_nnz"]
    assert SH.CAP == P["short_cap"]
    assert S.TILE == P["tile"] and S.LONG == P["long_row"]


# ------------------------------------------------------------------------------------------ emulations, bit for bit
EMU_PROFILES = ["lane_ends", "chunk_and_cta_borders", "long_row_edges", "tile_border_ends", "rows_cross_borders", "short_block_caps",
                "leading_trailing_empty", "nnz_zero", "one_row", "one_col", "rect_tall", "random_mix_0"]


def _fixture(profiles, name, kind):
    lens, cols = profiles[name]
    return E.Fixture(name, lens, cols, kind, seed=5)


@pytest.mark.parametrize("name", EMU_PROFILES)
@pytest.mark.parametrize("kind", ["f64", "wide"])
def test_flat_emulation_is_exact(P, profiles, name, kind):
    import test_flat_emulation as F
    f = _fixture(profiles, name, kind)
    for alpha, beta in E.SCALARS:
        y0 = f.y0f() if beta != 0 else np.full(f.rows, np.nan)
        got, written = F.emulate(f.off, f.col, f.val, f.xf(), y0, alpha, beta, warps=P["cta_nnz"] // P["warp_chunk"])
        assert np.all(written == 1)
        assert np.array_equal(got, f.want(alpha, beta)), (name, alpha, beta)


@pytest.mark.parametrize("name", EMU_PROFILES)
@pytest.mark.parametrize("seg_dense", [1, 24, 1000000])
def test_seg_emulation_is_exact(profiles, name, seg_dense):
    import test_seg_emulation as S
    f = _fixture(profiles, name, "wide")
    if f.nnz == 0:
        pytest.skip("the seg emulation starts from the tile partition of a matrix with non-zeros")
    for alpha, beta in E.SCALARS:
        y0 = f.y0f() if beta != 0 else np.full(f.rows, np.nan)
        got = S.emulate_spmv(f.off, f.col, f.val, f.xf(), y0, alpha, beta, seg_dense)[0]
        assert np.array_equal(got, f.want(alpha, beta)), (name, alpha, beta)


@pytest.mark.parametrize("name", EMU_PROFILES)
def test_short_emulation_is_exact(profiles, name):
    import test_short_emulation as SH
    f = _fixture(profiles, name, "wide")
    for alpha, beta in E.SCALARS:
        y0 = f.y0f() if beta != 0 else np.full(f.rows, np.nan)
        assert np.array_equal(SH.emulate(f.off, f.col, f.val, f.xf(), y0, alpha, beta), f.want(alpha, beta)), (name, alpha, beta)


# the host-compiled source of spmv_generic_kernels.cuh (the `emu` fixture of test_generic_emulation.py)
from test_generic_emulation import emu  # noqa: E402,F401  (pytest fixture)

A_DT = {"f32": 0, "f64": 1, "wide": 1, "mixed": 0}
XY_DT = {"f32": 0, "f64": 1, "wide": 1, "mixed": 1}
CT = {0: C.c_float, 1: C.c_double}
LL = C.c_longlong


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


GENERIC_PROFILES = ["lane_ends", "chunk_and_cta_borders", "long_row_edges", "short_block_caps", "leading_trailing_empty", "nnz_zero",
                    "one_row", "one_col", "rect_tall", "rect_wide"]


@pytest.mark.parametrize("kind", ["f32", "f64", "wide", "mixed"])
@pytest.mark.parametrize("base", [0, 1])
def test_generic_sources_are_exact(emu, profiles, kind, base):
    """csr_generic_kernel (every lane count, A and A^T), coo_generic_kernel (entries in random order) and sell_generic_kernel
    (slice sizes 1, 7, 32, 33; A and A^T) compiled for the host, on a grid of one CTA (several grid-stride trips)."""
    a_dt, xy_dt = A_DT[kind], XY_DT[kind]
    ct = CT[xy_dt]
    for name in GENERIC_PROFILES:
        f = _fixture(profiles, name, kind)
        off64, col64 = (f.off.astype(np.int64) + base), (f.col.astype(np.int64) + base)
        row64 = np.repeat(np.arange(f.rows, dtype=np.int64), np.diff(f.off)) + base
        perm = np.random.default_rng(9).permutation(f.nnz)
        for transpose in (0, 1):
            nx, ny = (f.rows, f.cols) if transpose else (f.cols, f.rows)
            x = E.values(kind, 0, nx, 0, 77)[1]
            y0 = E.values(kind, 0, 0, ny, 78)[2]
            xf, y0f = x.astype(E.NP_XY[kind]), y0.astype(E.NP_XY[kind])
            for alpha, beta in E.SCALARS:
                E.check_exact(f.off, f.col, f.a, x, y0, alpha, beta, 24 if xy_dt == 0 else 53, transpose=bool(transpose), cols=f.cols)
                want = E.reference(f.off, f.col, f.a, x, y0, alpha, beta, transpose=bool(transpose), cols=f.cols)
                fresh = lambda: y0f.copy() if beta != 0 else np.full(ny, np.nan, y0f.dtype)   # noqa: E731
                ca, cb = ct(alpha), ct(beta)
                for lanes_log2 in (0, 5):
                    y = fresh()
                    assert emu.emu_csr_generic(1, 1, a_dt, xy_dt, transpose, lanes_log2, 1, LL(f.rows), LL(f.cols), LL(f.nnz), _p(off64),
                                               _p(col64), _p(f.val), LL(base), C.byref(ca), C.byref(cb), _p(xf), _p(y)) == 0
                    assert np.array_equal(y, want), ("csr", name, transpose, lanes_log2, alpha, beta)
                y = fresh()
                r, c = (row64[perm], col64[perm]) if not transpose else (col64[perm], row64[perm])
                shape = (f.rows, f.cols) if not transpose else (f.cols, f.rows)
                assert emu.emu_coo_generic(1, a_dt, xy_dt, 1, LL(shape[0]), LL(shape[1]), LL(f.nnz), _p(r), _p(c),
                                           _p(np.ascontiguousarray(f.val[perm])), LL(base), C.byref(ca), C.byref(cb), _p(xf), _p(y)) == 0
                assert np.array_equal(y, want), ("coo", name, transpose, alpha, beta)
                for S in (1, 7, 32, 33):
                    so, sc, sv = O.csr_to_sell((f.off + base).astype(np.int32), (f.col + base).astype(np.int32), f.val, S, base=base)
                    y = fresh()
                    assert emu.emu_sell_generic(1, 1, a_dt, xy_dt, transpose, 1, LL(f.rows), LL(f.cols), LL(S), _p(so.astype(np.int64)),
                                                _p(sc.astype(np.int64)), _p(sv), LL(base), C.byref(ca), C.byref(cb), _p(xf), _p(y)) == 0
                    assert np.array_equal(y, want), ("sell", name, transpose, S, alpha, beta)


# ------------------------------------------------------------------------------------------ fused CG BLAS-1 (cg_fused.cu)
@pytest.fixture(scope="module")
def CGP(built_lib):
    return E.cg_params()


def test_cg_index_model_visits_every_element_once(CGP):
    """The model of the kernels' index mapping: every index in [0, n) is read exactly once (one 16-byte pair or the scalar
    tail), the scalar path runs at most once and only for odd n, and the grid never exceeds the cap."""
    for n in E.cg_sizes(CGP):
        w = E.cg_walk(n, CGP)
        assert np.array_equal(w["visits"], np.ones(n, np.int64)), n
        assert w["scalar_visits"] == n % 2, n
        assert 1 <= w["grid"] <= CGP["max_ctas"]
        assert w["passes"] == -(-n // (2 * w["grid"] * CGP["block"])), n


def test_cg_sizes_cover_every_class(CGP):
    hit = {}
    for n in E.cg_sizes(CGP):
        for c in E.cg_coverage(n, CGP):
            hit.setdefault(c, []).append(n)
    assert not set(E.CG_CLASSES) - set(hit), f"no size hits {sorted(set(E.CG_CLASSES) - set(hit))}"
    F = E.cg_full_pass(CGP)
    # the sizes sit on the kernels' borders: the first size at the grid cap, F itself, F + 1
    first_at_cap = min(hit["cap_single_pass"])
    assert E.cg_grid(first_at_cap, CGP) == CGP["max_ctas"] and E.cg_grid(first_at_cap - 2, CGP) == CGP["max_ctas"] - 1
    assert hit["exactly_one_full_pass"] == [F] and F + 1 in hit["odd_tail_later_pass_at_cap"]
    assert max(E.cg_walk(n, CGP)["passes"] for n in E.cg_sizes(CGP)) >= 4


def test_cg_coverage_notices_a_missing_class(CGP):
    """Without the sizes that carry them, classes go missing: the coverage check is not vacuous."""
    P2, F = 2 * CGP["block"], E.cg_full_pass(CGP)
    hit = set()
    for n in E.cg_sizes(CGP):
        if n not in (1, P2 + 1, 2 * P2 + 1, 5 * P2 + 1, F):
            hit |= E.cg_coverage(n, CGP)
    assert {"scalar_tail_only", "odd_tail_later_pass_below_cap", "exactly_one_full_pass"} <= set(E.CG_CLASSES) - hit


@pytest.mark.parametrize("kind", E.CG_KINDS)
def test_cg_reference_is_exact_at_every_size(CGP, kind):
    """The precondition (asserted inside cg_reference) holds at every size up to the largest, and the reference agrees with
    float64 numpy on the operations where float64 is exact too."""
    for name, k in E.CG_KERNELS.items():
        for n in E.cg_sizes(CGP):
            v = E.cg_vectors(kind, n, k.vectors, seed=n)
            want = E.cg_reference(name, v)
            assert set(want) == set(k.writes) | ({k.reduces} if k.reduces else set())
            f = {key: a.astype(np.float64) for key, a in v.items()}
            if "x" in want:
                assert np.array_equal(want["x"], f["x"] + (-0.25) * f["p"])
            if "p" in want:
                assert np.array_equal(want["p"], f["r"] + 0.5 * f["p"])
            if "r" in want:
                assert np.array_equal(want["r"], f["r"] - (-0.25) * f["t"])
                assert want["delta_new"] == math.fsum(want["r"] * want["r"])
            if name == "dot":
                assert want["out"] == math.fsum(f["a"] * f["b"])


def test_cg_wide_vectors_need_more_than_fp32(CGP):
    """At the largest size an fp32 accumulator loses bits on both kinds; the "wide" products alone need more than 24 bits."""
    n = E.cg_sizes(CGP)[-1]
    for kind in E.CG_KINDS:
        v = E.cg_vectors(kind, n, ["a", "b"], seed=1)
        assert np.abs(v["a"] * v["b"]).sum() > 1 << 24
    v = E.cg_vectors("wide", 1000, ["a", "b"], seed=1)
    assert np.abs(v["a"] * v["b"]).min() >= 1 << 24
    assert np.all(v["a"] != 0) and np.all(E.cg_vectors("f64", 1000, ["a"], seed=2)["a"] != 0)
