// config.h -- run-time switches of libb200spmv.so, read from the environment ONCE (first use) and changeable
// afterwards only through b200spmv_set_option() (tests / tuning sweeps).  Nothing on the launch path calls getenv().
#pragma once

namespace b200 {

struct Config {
    int csr_kernel  = -1;   // B200SPMV_CSR_KERNEL = tile|pipe|ws|rowwise|seg ; -1 = run-time choice
    int tile_scatter = 0;   // B200SPMV_TILE_ORDER = scatter
    int pdl         = 0;    // B200SPMV_PDL = 1: launch the CSR fix-up kernel with programmatic stream serialization
    int seg_dense   = 24;   // B200SPMV_SEG_DENSE: csr_seg_kernel takes the register path for tiles with >= this many nnz per row
    int sell_generic = 0;   // B200SPMV_SELL_GENERIC = 1: never use the slice-32 specialisation
    int flat        = -1;   // B200SPMV_FLAT = auto|on|off: the preprocess-built flat CSR plan (csr_flat_kernel); auto = by the matrix' row statistic
    int flat_quiet_permille = 350;   // B200SPMV_FLAT_QUIET: auto picks the flat kernel when at least this share of the 32-non-zero steps ends no row
    int short_rows  = -1;   // B200SPMV_SHORT = auto|on|off: csr_short_kernel (warp per 32 rows); auto = preprocess found no row longer than 32
    int coo_kernel  = -1;   // B200SPMV_COO_KERNEL = tile|seg ; -1 = default (seg)
    int generic     = 1;    // B200SPMV_GENERIC = off|csr|all: what spmv_generic.cu serves instead of the closed library.
                            //   csr (default): CSR with 64-bit indices / fp32 A with fp64 vectors / their transposes / no buffer --
                            //                  validated on the GPU by tests/test_generic_gpu.py;
                            //   all: also COO and Sliced-ELL of those kinds, Sliced-ELL transposes, strided-batch SpMM -- written
                            //        and emulated on the CPU, their first hardware run is tests/test_zz_unverified_gpu.py;
                            //   off: everything of that kind goes to the closed library
    int zcsr        = 0;    // B200SPMV_ZCSR = auto|on: cusparseSpMV on a double-complex CSR A.  auto (0, default): b200spmv_csr_z
                            //   only in the classes measured at least at parity (none today, DESIGN.md 3.21); on (1): every call
                            //   in b200spmv_csr_z's class
    int dense       = 0;    // B200SPMV_DENSE = auto|on: cusparseSparseToDense / cusparseDenseToSparse_convert.  auto (0, default):
                            //   the native kernels only in the classes measured at least at parity (DESIGN.md 3.24); on (1): every
                            //   call b200dense_route admits, so the shim's native path can be exercised before a measurement routes it
    int banded      = 0;    // B200SPMV_BANDED = auto|on: cusparse<t>gpsvInterleavedBatch / gtsvInterleavedBatch.  auto (0, default):
                            //   the native solves only in the classes measured at least at parity (DESIGN.md 3.25); on (1): every
                            //   call b200banded_route admits
    int ilu0        = 0;    // B200SPMV_ILU0 = auto|on: cusparse<t>csrilu02 / csric02.  auto (0, default): the native factorization only
                            //   in the classes measured at least at parity (DESIGN.md 3.26); on (1): every call b200ilu0_route admits
    int spgemm      = 0;    // B200SPMV_SPGEMM = auto|on: cusparseSpGEMMreuse_compute.  auto (0, default): the native numeric phase only
                            //   in the classes measured at least at parity (DESIGN.md 3.28); on (1): every call b200spgemm_route admits
};

Config& config();

// counters a test can read: how many SpMV calls ran on our kernels / were handed to the closed library
struct Stats {
    unsigned long long native_calls = 0, forwarded_calls = 0, analyze_calls = 0;
    const char* last_csr_kernel = "none";   // name of the main kernel of the most recent CSR launch
};
Stats& stats();

}  // namespace b200
