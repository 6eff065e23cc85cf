"""CPU: the C-ABI library builds for sm_90a, loads, and exports every symbol include/b200spmv.h declares."""
import ctypes
import os
import re
import subprocess

import pytest

from cudalibrarysamples_b200 import build
from cudalibrarysamples_b200.lib import load, prototypes, signatures

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def declared_symbols(header="b200spmv.h"):
    return sorted({name for _, name, _ in prototypes(header)})


def exported(lib):
    out = subprocess.check_output(["nm", "-D", "--defined-only", lib], text=True)
    return {line.split()[-1] for line in out.splitlines() if " T " in line}


def test_header_declares_the_reference_entry_points():
    names = declared_symbols()
    # the exact symbols the reference's SpMV samples bind (SURVEY.md 8b)
    for n in ["cusparseCreateCsr", "cusparseCreateConstCsr", "cusparseCreateCoo", "cusparseCreateSlicedEll",
              "cusparseCreateDnVec", "cusparseDestroySpMat", "cusparseDestroyDnVec", "cusparseSpMV_bufferSize",
              "cusparseSpMV_preprocess", "cusparseSpMV", "cusparseCsrSetPointers", "cusparseDnVecSetValues",
              "b200spmv_csr_mv", "b200spmv_coo_mv", "b200spmv_sell_mv", "b200spmv_csr_analyze"]:
        assert n in names, n


def test_library_exports_every_declared_symbol(built_lib):
    have = exported(built_lib)
    missing = [n for n in declared_symbols() if n not in have]
    assert not missing, missing


def test_bench_plumbing_is_not_part_of_the_product_abi(built_lib):
    """The synthetic-workload generators live in libb200gen.so (include/b200gen.h); libb200spmv.so exports none of them."""
    assert not [n for n in exported(built_lib) if n.startswith("b200gen")]
    assert not [n for n in declared_symbols() if n.startswith("b200gen")]
    gen = declared_symbols("b200gen.h")
    assert len(gen) >= 6
    have = exported(build.GEN_LIB_PATH)
    assert not [n for n in gen if n not in have]


def test_options_are_set_through_the_abi_not_the_environment(built_lib):
    lib = load(built_lib)
    assert lib.b200spmv_set_option(b"B200SPMV_CSR_KERNEL", b"seg") == 0
    assert lib.b200spmv_set_option(b"B200SPMV_CSR_KERNEL", b"auto") == 0
    assert lib.b200spmv_set_option(b"B200SPMV_CSR_KERNEL", b"no-such-kernel") == -1
    assert lib.b200spmv_set_option(b"NO_SUCH_KEY", b"1") == -1
    for v in (b"off", b"all", b"csr"):                      # what spmv_generic.cu serves; "csr" is the default
        assert lib.b200spmv_set_option(b"B200SPMV_GENERIC", v) == 0
    assert lib.b200spmv_set_option(b"B200SPMV_GENERIC", b"everything") == -1
    n, f, a = ctypes.c_uint64(7), ctypes.c_uint64(7), ctypes.c_uint64(7)
    lib.b200spmv_reset_stats()
    lib.b200spmv_get_stats(ctypes.byref(n), ctypes.byref(f), ctypes.byref(a))
    assert (n.value, f.value, a.value) == (0, 0, 0)
    # no getenv on the launch path: the only getenv calls of the library sit in the once-only initialisers
    src = os.path.join(ROOT, "cudalibrarysamples_b200", "csrc")
    for name in ("spmv_csr.cu", "spmv_coo_sell.cu"):
        assert "getenv(" not in open(os.path.join(src, name)).read(), name


def test_library_loads_without_a_gpu(built_lib):
    lib = load(built_lib)
    assert b"sm_90a" in lib.b200spmv_version()
    t, l, b = ctypes.c_int32(), ctypes.c_int32(), ctypes.c_int32()
    lib.b200spmv_csr_plan_params(ctypes.byref(t), ctypes.byref(l), ctypes.byref(b))
    assert t.value > l.value > 0 and b.value % 32 == 0
    nt = lib.b200spmv_csr_num_tiles(ctypes.c_int64(1000), ctypes.c_int64(16000))
    assert nt == (17000 + t.value - 1) // t.value
    ws = lib.b200spmv_csr_workspace_bytes(ctypes.c_int64(1000), ctypes.c_int64(16000))
    assert ws >= (nt + 1) * (8 + 4 + 8 + 8)
    # the CG workspace: one partial sum per CTA of the largest grid, then the arrival counter in its own 8-byte slot (+ 1 spare)
    blk, max_ctas = ctypes.c_int32(), ctypes.c_int32()
    lib.b200cg_params(ctypes.byref(blk), ctypes.byref(max_ctas))
    assert blk.value % 32 == 0 and max_ctas.value > 0
    assert lib.b200cg_workspace_bytes() == (max_ctas.value + 2) * 8
    # argument validation happens on the host, before any CUDA call
    assert lib.b200spmv_csr_mv(None, 7, ctypes.c_int64(4), ctypes.c_int64(4), ctypes.c_int64(9), None, None, None, 0,
                               None, None, 0, None, None, None) == -1


HEADERS = [("b200spmv.h", build.LIB_PATH), ("b200spsv.h", build.SPSV_LIB_PATH), ("b200gen.h", build.GEN_LIB_PATH)]


@pytest.mark.parametrize("header", [h for h, _ in HEADERS])
def test_every_b200_prototype_has_a_ctypes_signature(header):
    """each B200*_EXPORT tag of the header starts a prototype the parser reads, and every b200* one maps to ctypes types"""
    with open(os.path.join(ROOT, "include", header)) as f:
        text = re.sub(r"/\*.*?\*/", " ", f.read(), flags=re.S)
    tags = len(re.findall(r"\bB200\w*_EXPORT\b", text)) - 1                # minus its #define
    assert len(prototypes(header)) == tags
    assert sorted(signatures(header)) == [n for n in declared_symbols(header) if n.startswith("b200")]


@pytest.mark.parametrize("header, path", HEADERS)
def test_declared_and_exported_b200_functions_are_the_same(built_lib, header, path):
    load(path, header=header)                                                # resolves every declared name, or raises
    assert {n for n in exported(path) if n.startswith("b200")} == set(signatures(header))


def test_signatures_follow_the_header():
    spmv, gen = signatures("b200spmv.h"), signatures("b200gen.h")
    i32, i64 = ctypes.c_int, ctypes.c_int64
    assert spmv["b200spmv_csr_workspace_bytes"] == (ctypes.c_size_t, [i64, i64])
    assert spmv["b200spmv_version"] == (ctypes.c_char_p, [])
    assert gen["b200gen_stencil5_fill"][1][2:5] == [ctypes.c_double] * 3
    assert spmv["b200spmm_coo_workspace_bytes"] == (ctypes.c_size_t, [i32, i32, i64, i64, i64, i64, i32, i32, i64])


def test_declarations_are_live(built_lib):
    lib = load(built_lib)
    with pytest.raises(ctypes.ArgumentError):                                # an int64_t where the header says int
        lib.b200spmm_coo_workspace_bytes(ctypes.c_int64(0), 0, 100, 80, 8, 1000, 1, 1, 0)
    nnz = 1 << 40                                                            # plain ints, a size_t result past 2^32
    nt = lib.b200spmv_csr_num_tiles(1000, nnz)
    ws = lib.b200spmv_csr_workspace_bytes(1000, nnz)
    assert ws > 1 << 32 and ws >= (nt + 1) * (8 + 4 + 8 + 8)


def test_only_lib_py_declares_native_signatures():
    """every b200* signature comes from lib.load(); the checker's own oracle library declares its few functions itself"""
    allowed = {os.path.join("cudalibrarysamples_b200", "lib.py"), os.path.join("oracle", "oracle.py")}
    found = []
    for d, dirs, files in os.walk(ROOT):
        dirs[:] = [x for x in dirs if not x.startswith(".") and x != "__pycache__"]
        for name in files:
            rel = os.path.relpath(os.path.join(d, name), ROOT)
            if name.endswith(".py") and rel not in allowed:
                with open(os.path.join(d, name)) as f:
                    found += [f"{rel}:{i}" for i, line in enumerate(f, 1) if re.search(r"\b(argtypes|restype)\s*=(?!=)", line)]
    assert not found, found


def kernel_sass(built_lib, pattern):
    sass = subprocess.check_output(["cuobjdump", "-sass", built_lib], text=True)
    assert "arch = sm_90a" in sass
    m = re.search(r"Function : \S*" + pattern + r".*?(?=Function :|\Z)", sass, re.S)
    assert m, pattern + " not found in the cubin"
    return m.group(0)


def test_sass_of_the_seg_kernel(built_lib):
    """What the selectable csr_seg_kernel<double> (register accumulation + segmented scan per tile) really emits: 64-bit L1-no-allocate streaming
    loads of val[] (lane-consecutive: 256 B per warp instruction -- per-lane 128-bit loads were measured slower, see
    DESIGN.md), 32-bit ones of col_ind[], x through the read-only path, shuffle / vote / redux based row reduction, no
    tensor cores.  profiles/sass_summary_r2.md holds the per-kernel instruction counts."""
    body = kernel_sass(built_lib, "csr_seg_kernelId")
    assert re.search(r"LDG\.E\.NA\.64", body)          # val[]: ld.global.nc.L1::no_allocate.f64
    assert re.search(r"LDG\.E\.NA(?!\.64)", body)      # col_ind[]: 32-bit no-allocate
    assert re.search(r"LDG\.E\.64\.CONSTANT", body)   # x gathered through the read-only L1 path
    assert "SHFL" in body and "VOTE" in body and "REDUX" in body
    assert not re.search(r"LDG\.E\S*\.128", body)      # no 128-bit per-lane loads in this kernel
    assert "HMMA" not in body and "UTC" not in body and "UTMA" not in body   # no tensor cores, no tensor-map TMA


def test_sass_of_the_headline_kernel(built_lib):
    """csr_flat_kernel<double> -- what bench.py's headline number runs on (profiles/sass_summary_r2.md has the full table):
    the val[] / col_ind[] streams as 64- / 32-bit L1-no-allocate loads (lane-consecutive: 256 B / 128 B per warp instruction),
    x gathered through the read-only path, butterfly + segmented-scan shuffles, no per-lane 128-bit global loads, a CTA
    barrier only at the stitch, no bulk copies, no tensor cores."""
    body = kernel_sass(built_lib, "csr_flat_kernelId")
    assert len(re.findall(r"LDG\.E\.NA\.64", body)) == 8 and len(re.findall(r"LDG\.E\.NA\.CONSTANT", body)) == 8   # 8 steps of 32 per warp chunk
    assert re.search(r"LDG\.E\.64\.CONSTANT", body)
    assert "SHFL.BFLY" in body and "SHFL.UP" in body and "VOTE" in body
    assert not re.search(r"LDG\.E\S*\.128", body)
    assert len(re.findall(r"\bBAR\.", body)) <= 3
    assert "UBLKCP" not in body and "HMMA" not in body and "UTC" not in body and "UTMA" not in body


def test_sass_summary_in_profiles_is_current(built_lib):
    """profiles/sass_summary_r2.md is generated from the built library (scripts/sass_summary.py): the committed table must list
    every kernel the library contains."""
    table = open(os.path.join(ROOT, "profiles", "sass_summary_r2.md")).read()
    sass = subprocess.check_output(["cuobjdump", "-sass", built_lib], text=True)
    kernels = set(re.findall(r"Function : _ZN\d+b200(?:cg|peer)?\d+([a-z0-9_]+_kernel)", sass))     # _ZN4b20015csr_flat_kernelIdE... -> csr_flat_kernel
    assert kernels and not [k for k in kernels if k not in table]


def test_sass_of_the_tma_fed_variant(built_lib):
    body = kernel_sass(built_lib, "csr_ws_kernelId")
    assert "UBLKCP" in body and "SYNCS" in body         # cp.async.bulk + mbarrier


def test_reference_samples_bind_spmv_to_the_shim():
    """oracle/_ref/*.b200 are the unmodified reference samples linked `-lb200spmv -lcusparse` (oracle/Makefile)."""
    exe = os.path.join(ROOT, "oracle", "_ref", "cg_example.b200")
    if not os.path.exists(exe):
        import pytest
        pytest.skip("oracle/_ref not built (needs /root/reference)")
    env = dict(os.environ, LD_BIND_NOW="1", LD_DEBUG="bindings")
    p = subprocess.run([exe], env=env, capture_output=True, text=True)
    lines = [l for l in p.stderr.splitlines() if "cg_example.b200 [0] to" in l]
    def target(sym):
        return [l for l in lines if f"`{sym}'" in l][0]
    assert "libb200spmv.so" in target("cusparseSpMV")
    assert "libb200spmv.so" in target("cusparseCreateCsr")
    assert "libcusparse.so.12" in target("cusparseSpSV_solve")
    assert "libcusparse.so.12" in target("cusparseCreate")


def test_ld_preload_rebinds_an_already_built_sample():
    """INTEGRATION.md section 2: the stock binary (linked against the real libcusparse only) picks up the shim's SpMV
    symbols under LD_PRELOAD; everything else stays with the closed library."""
    exe = os.path.join(ROOT, "oracle", "_ref", "spmv_csr_example.cusparse")
    lib = os.path.join(ROOT, "cudalibrarysamples_b200", "libb200spmv.so")
    if not (os.path.exists(exe) and os.path.exists(lib)):
        import pytest
        pytest.skip("oracle/_ref or the library not built")
    env = dict(os.environ, LD_BIND_NOW="1", LD_DEBUG="bindings", LD_PRELOAD=lib)
    p = subprocess.run([exe], env=env, capture_output=True, text=True)
    lines = [l for l in p.stderr.splitlines() if "spmv_csr_example.cusparse [0] to" in l]
    def target(sym):
        return [l for l in lines if f"`{sym}'" in l][0]
    for sym in ("cusparseSpMV", "cusparseSpMV_bufferSize", "cusparseSpMV_preprocess", "cusparseCreateCsr", "cusparseCreateDnVec"):
        assert "libb200spmv.so" in target(sym), sym
    assert "libcusparse.so.12" in target("cusparseCreate")
