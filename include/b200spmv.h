/*
 * b200spmv.h -- C ABI of libb200spmv.so, the H100-native (sm_90a) drop-in for the cusparseSpMV path
 * of NVIDIA/CUDALibrarySamples (cuSPARSE/spmv_csr, spmv_coo, spmv_sell, cg, bicgstab).
 *
 * Two layers, both `extern "C"`, plain pointers and sizes only:
 *
 *   1. The cuSPARSE generic-API symbols the samples call.  The shim re-exports them with the exact
 *      prototypes of the CUDA 12.9 toolkit header the samples include
 *      (cuSPARSE/spmv_csr/spmv_csr_example.c:19 `#include <cusparse.h>`); every other cusparse* symbol
 *      keeps resolving to the real libcusparse.so.12 (link order `-lb200spmv -lcusparse`, or LD_PRELOAD).
 *
 *   2. The native entry points underneath (b200spmv_*): descriptor-free, usable without libcusparse.
 *
 * Every function the library exports is tagged B200SPMV_EXPORT; tests/test_abi.py greps this header for
 * the tag and checks that each symbol is present in the built .so.
 */
#ifndef B200SPMV_H_
#define B200SPMV_H_

#include <stddef.h>
#include <stdint.h>

#define B200SPMV_EXPORT /* exported from libb200spmv.so */

#ifdef __cplusplus
extern "C" {
#endif

/* ============================================================================================== *
 * Layer 2: native entry points.                                                                   *
 *   stream    : cudaStream_t (passed as void*); all work is enqueued asynchronously on it, no     *
 *               host synchronisation, no allocation -> CUDA-graph capturable.                     *
 *   dtype     : 0 = fp32 (== CUDA_R_32F), 1 = fp64 (== CUDA_R_64F); A, x, y and the arithmetic    *
 *               all use this type.  Indices are int32.  base is 0 or 1.                           *
 *   alpha/beta: pointers to one value of `dtype`; host memory when scalars_on_device == 0,        *
 *               device memory (read inside the kernel) otherwise.                                 *
 *   return    : 0 on success, -1 on invalid arguments, otherwise the cudaError_t of the launch.   *
 * ============================================================================================== */

/* CSR.  The workspace holds the structure-only tile partition ("plan") built by _analyze:
 * replaces cusparseSpMV_bufferSize / cusparseSpMV_preprocess / cusparseSpMV for
 * cusparseCreateCsr descriptors (cuSPARSE/spmv_csr/spmv_csr_example.c:97-112,
 * cuSPARSE/cg/cg_example.c:409-418,156-160,220-224,294-297). */
B200SPMV_EXPORT size_t b200spmv_csr_workspace_bytes(int64_t rows, int64_t nnz);
B200SPMV_EXPORT int    b200spmv_csr_analyze(void* stream, int64_t rows, int64_t nnz, const void* row_offsets,
                                            int32_t base, void* workspace);
B200SPMV_EXPORT int    b200spmv_csr_mv(void* stream, int dtype, int64_t rows, int64_t cols, int64_t nnz,
                                       const void* row_offsets, const void* col_ind, const void* values,
                                       int32_t base, const void* alpha, const void* beta, int scalars_on_device,
                                       const void* x, void* y, void* workspace);
/* Introspection used by the parity tests (bit-exact integer preprocessing): number of tiles, and the
 * constants the partition was built with. */
B200SPMV_EXPORT int64_t b200spmv_csr_num_tiles(int64_t rows, int64_t nnz);
B200SPMV_EXPORT void    b200spmv_csr_plan_params(int32_t* tile_items, int32_t* long_row, int32_t* block_threads);
B200SPMV_EXPORT size_t  b200spmv_csr_plan_tiles_offset(void);
/* byte offsets inside the workspace of the control words {finished CTAs, number of split rows} and of the split-row
 * list (int4 {row, first covering tile, last covering tile, 0}) */
B200SPMV_EXPORT size_t  b200spmv_csr_plan_ctl_offset(int64_t rows, int64_t nnz);
B200SPMV_EXPORT size_t  b200spmv_csr_plan_split_offset(int64_t rows, int64_t nnz);

/* CSR, "flat" plan (spmv_csr_flat.cu): a second, larger structure-only plan -- one bit per non-zero marking row ends, a
 * run counter per 256 non-zeros, the list of non-empty rows, and the hot-column copy of col_ind below -- built once by cusparseSpMV_preprocess for matrices with
 * long / skewed rows; the SpMV kernel then needs no row offsets, no shared-memory staging and no barriers inside a warp's
 * chunk.  Same call sites as above (spmv_csr_example.c:104-112: preprocess, then SpMV). */
B200SPMV_EXPORT size_t b200spmv_csr_flat_workspace_bytes(int64_t rows, int64_t nnz);
B200SPMV_EXPORT int    b200spmv_csr_flat_analyze(void* stream, int64_t rows, int64_t nnz, const void* row_offsets,
                                                 int32_t base, void* workspace);
/* The hot-column part of the flat plan, built after _flat_analyze in the same workspace (needs cols <= nnz rounded up to
 * 2048, else no hot plan).  The hot columns are those used at least tau times, tau >= 2 the smallest threshold whose columns
 * fit b200spmv_csr_flat_hot_params' byte budget for this dtype; they get slots 0..H-1 in ascending column order.  colp
 * (int32 per non-zero, 0 behind nnz up to the padded chunk count) holds ~slot for a hot column, else the 0-based column.
 * H = 0 when the hot columns take less than min_share_permille / 1000 of nnz, or while the stream is being captured.
 * Reads a column-count histogram back: synchronises the stream once.  *hot_out = H, to be passed to _flat_mv; the
 * workspace's control words (see _flat_plan_offsets) hold H at [4] and tau at [5].  The plan depends on col_ind only, so
 * it stays valid when the values change. */
B200SPMV_EXPORT int    b200spmv_csr_flat_hot_analyze(void* stream, int dtype, int64_t rows, int64_t cols, int64_t nnz,
                                                     const void* col_ind, int32_t base, void* workspace, int32_t* hot_out);
B200SPMV_EXPORT void   b200spmv_csr_flat_hot_offsets(int64_t rows, int64_t nnz, size_t* colp, size_t* hot);
B200SPMV_EXPORT void   b200spmv_csr_flat_hot_params(int32_t* hot_bytes, int32_t* min_share_permille, int32_t* bins);
/* hot: the H of b200spmv_csr_flat_hot_analyze, or 0 (the kernel then reads col_ind).  With H > 0 a small kernel first
 * packs x[hot[j]] into the workspace and csr_flat_kernel reads colp: the same products in the same order, so y is
 * bit-identical to the H = 0 call. */
B200SPMV_EXPORT int    b200spmv_csr_flat_mv(void* stream, int dtype, int64_t rows, int64_t cols, int64_t nnz,
                                            const void* row_offsets, const void* col_ind, const void* values,
                                            int32_t base, const void* alpha, const void* beta, int scalars_on_device,
                                            const void* x, void* y, void* workspace, int32_t hot);
/* byte offsets of the flat plan's arrays inside its workspace: endmask (uint32 per 32 non-zeros, zero-padded to a
 * multiple of 64 words), chunk_run (int32 per 256 non-zeros, padded to whole groups of 8, + 1), nzrow (int32, rows + 2), control words
 * {non-empty rows, steps without a row end, steps} -- read back by the bit-exact preprocessing tests */
B200SPMV_EXPORT void   b200spmv_csr_flat_plan_offsets(int64_t rows, int64_t nnz, size_t* endmask, size_t* chunk_run,
                                                      size_t* nzrow, size_t* ctl);
/* the constants csr_flat_kernel was built with: non-zeros per warp chunk, per CTA, and per chunk_run entry of the plan
 * (the exact-arithmetic tests place row ends around these borders) */
B200SPMV_EXPORT void   b200spmv_csr_flat_params(int32_t* warp_chunk, int32_t* cta_nnz, int32_t* plan_chunk);

/* CSR, all rows short (spmv_csr_short.cu): a warp per 32 consecutive rows, products staged in the warp's own slice of
 * shared memory, one lane per row adds them up; needs no plan, only the caller's row offsets.  cusparseSpMV_preprocess picks
 * it when the longest row (b200spmv_csr_max_row_length, written to device memory) has at most b200spmv_csr_short_max_row()
 * non-zeros -- the stencil operators of cuSPARSE/cg/cg_example.c:71-128 and cuSPARSE/bicgstab/bicgstab_example.c:69-127. */
B200SPMV_EXPORT int    b200spmv_csr_short_max_row(void);
/* csr_short_kernel's constants: products one warp stages per pass (SHORT_CAP), rows per warp */
B200SPMV_EXPORT void   b200spmv_csr_short_params(int32_t* pass_cap, int32_t* rows_per_warp);
B200SPMV_EXPORT int    b200spmv_csr_max_row_length(void* stream, int64_t rows, const void* row_offsets, int32_t* out_device);
B200SPMV_EXPORT int    b200spmv_csr_short_mv(void* stream, int dtype, int64_t rows, int64_t cols, int64_t nnz,
                                             const void* row_offsets, const void* col_ind, const void* values,
                                             int32_t base, const void* alpha, const void* beta, int scalars_on_device,
                                             const void* x, void* y);

/* The same product with a dot product in its epilogue: *dot_out = y . w, fp64 accumulation, deterministic (SURVEY.md 8(f)-2:
 * T = A*P and T . P of cg_example.c:220-227 in one pass).  dot_out: device memory.  workspace:
 * b200spmv_csr_short_dot_workspace_bytes() bytes, zeroed once before its first use. */
B200SPMV_EXPORT size_t b200spmv_csr_short_dot_workspace_bytes(void);
B200SPMV_EXPORT int    b200spmv_csr_short_mv_dot(void* stream, int dtype, int64_t rows, int64_t cols, int64_t nnz,
                                                 const void* row_offsets, const void* col_ind, const void* values,
                                                 int32_t base, const void* alpha, const void* beta, int scalars_on_device,
                                                 const void* x, void* y, const void* w, double* dot_out, void* workspace);

/* CSR, opA = TRANSPOSE (spmv_csr_transpose.cu): y[cols] = alpha * A^T * x[rows] + beta * y; no plan, no workspace; one
 * fp atomic per non-zero, so the summation order (not the tolerance) differs between runs. */
B200SPMV_EXPORT int    b200spmv_csr_transpose_mv(void* stream, int dtype, int64_t rows, int64_t cols, int64_t nnz,
                                                 const void* row_offsets, const void* col_ind, const void* values,
                                                 int32_t base, const void* alpha, const void* beta, int scalars_on_device,
                                                 const void* x, void* y);

/* CSR x dense: C = alpha*A*B + beta*C, A rows x cols (CSR, int32 indices), B cols x n, C rows x n, each dense matrix row- or
 * column-major with leading dimension ld* (elements).  Replaces cusparseSpMM for CSR descriptors, opA = opB = NON_TRANSPOSE
 * (cuSPARSE/spmm_csr/spmm_csr_example.c:105-132).  b200spmm_csr needs no workspace; b200spmm_csr_ws takes one of
 * b200spmm_csr_workspace_bytes() bytes (what cusparseSpMM_bufferSize reports, spmm_csr_example.c:105-110) and uses it for a
 * row-major copy of a column-major B -- the sample's own layout then runs at the row-major speed. */
B200SPMV_EXPORT size_t b200spmm_csr_workspace_bytes(int dtype, int64_t cols, int64_t n, int b_row_major);
B200SPMV_EXPORT int b200spmm_csr_ws(void* stream, int dtype, int64_t rows, int64_t cols, int64_t n, int64_t nnz,
                                    const void* row_offsets, const void* col_ind, const void* values, int32_t base,
                                    const void* alpha, const void* beta, int scalars_on_device, const void* B, int64_t ldb,
                                    int b_row_major, void* C, int64_t ldc, int c_row_major, void* workspace);
B200SPMV_EXPORT int b200spmm_csr(void* stream, int dtype, int64_t rows, int64_t cols, int64_t n, int64_t nnz,
                                 const void* row_offsets, const void* col_ind, const void* values, int32_t base,
                                 const void* alpha, const void* beta, int scalars_on_device, const void* B, int64_t ldb,
                                 int b_row_major, void* C, int64_t ldc, int c_row_major);

/* The BLAS-1 part of a CG iteration, fused, all scalars in DEVICE memory (no host synchronisation, CUDA-graph capturable).
 * Replaces the cublasDdot / cublasDaxpy / cublasDnrm2 / cublasDscal calls between two cusparseSpMV calls of gpu_CG
 * (cuSPARSE/cg/cg_example.c:226-286).  fp64; vectors 16-byte aligned; `workspace` = b200cg_workspace_bytes() bytes, zeroed
 * once by the caller.
 *   b200cg_dot        *out = a . b
 *   b200cg_update_xr  alpha = *delta / *denom;  x += alpha p;  r -= alpha t;  *delta_new = r . r   (one pass)
 *   b200cg_update_p   beta = *delta_new / *delta;  p = r + beta p
 * Every kernel walks the vectors in pairs (16-byte loads, a scalar tail for odd n) with a grid-stride loop over
 * min(ceil((n / 2) / block), max_ctas) CTAs of `block` threads; the workspace holds max_ctas partial sums, then the arrival
 * counter (uint32 at byte max_ctas * 8), which every reduction leaves at zero.  b200cg_params reports block and max_ctas
 * (the exact-arithmetic tests size their vectors around these borders). */
B200SPMV_EXPORT size_t b200cg_workspace_bytes(void);
B200SPMV_EXPORT void   b200cg_params(int32_t* block, int32_t* max_ctas);
B200SPMV_EXPORT int    b200cg_dot(void* stream, int64_t n, const double* a, const double* b, double* out, void* workspace);
B200SPMV_EXPORT int    b200cg_update_xr(void* stream, int64_t n, double* x, double* r, const double* p, const double* t,
                                        const double* delta, const double* denom, double* delta_new, void* workspace);
/*   b200cg_update_r   alpha = *delta / *denom;  r -= alpha t;  *delta_new = r . r            (x is not touched)
 *   b200cg_update_xp  x += alpha p;  beta = *delta_new / *delta;  p = r + beta p              (p read once)
 * A CG iteration of b200cg_dot + _update_r + _update_xp reads or writes a whole vector 10 times (2 + 3 + 5); with _update_xr +
 * _update_p instead it is 11 (2 + 6 + 3). */
B200SPMV_EXPORT int    b200cg_update_r(void* stream, int64_t n, double* r, const double* t, const double* delta, const double* denom,
                                       double* delta_new, void* workspace);
B200SPMV_EXPORT int    b200cg_update_xp(void* stream, int64_t n, double* x, double* p, const double* r, const double* delta,
                                        const double* denom, const double* delta_new);
B200SPMV_EXPORT int    b200cg_update_p(void* stream, int64_t n, double* p, const double* r, const double* delta_new,
                                       const double* delta);

/* Device-side barrier over NVLink peer memory (one process per GPU, one box), graph-replay safe: the epoch lives in device
 * memory.  peer_flag_ptrs_dev: device array of `world` pointers, entry r = rank r's flag array (`world` 8-byte slots,
 * zero-initialised, mapped into this process: symmetric memory / CUDA IPC); epoch_dev: one zero-initialised 8-byte counter
 * in local device memory.  A rank that does not arrive within timeout_seconds makes the kernel trap (CUDA error). */
B200SPMV_EXPORT int b200peer_barrier(void* stream, const void* peer_flag_ptrs_dev, void* epoch_dev, int my_rank, int world,
                                     double timeout_seconds);
/* dst[0, bytes) = src[0, bytes) with `ctas` CTAs of 256 threads, 16-byte loads / stores (both pointers 16-byte aligned):
 * the SM-side pull of a peer's x shard over NVLink. */
B200SPMV_EXPORT int b200peer_pull(void* stream, void* dst, const void* src, size_t bytes, int ctas);

/* COO (row-sorted or not).  Replaces cusparseSpMV for cusparseCreateCoo descriptors
 * (cuSPARSE/spmv_coo/spmv_coo_example.c:86-104). */
B200SPMV_EXPORT size_t b200spmv_coo_workspace_bytes(int64_t rows, int64_t nnz);
B200SPMV_EXPORT int    b200spmv_coo_mv(void* stream, int dtype, int64_t rows, int64_t cols, int64_t nnz,
                                       const void* row_ind, const void* col_ind, const void* values,
                                       int32_t base, const void* alpha, const void* beta, int scalars_on_device,
                                       const void* x, void* y, void* workspace);

/* Sliced-ELL.  Replaces cusparseSpMV for cusparseCreateSlicedEll descriptors
 * (cuSPARSE/spmv_sell/spmv_sell_example.c:103-122).  Padding entries have column index -1 (+base). */
B200SPMV_EXPORT size_t b200spmv_sell_workspace_bytes(int64_t rows, int64_t sell_values_size, int64_t slice_size);
B200SPMV_EXPORT int    b200spmv_sell_mv(void* stream, int dtype, int64_t rows, int64_t cols, int64_t slice_size,
                                        const void* slice_offsets, const void* col_ind, const void* values,
                                        int32_t base, const void* alpha, const void* beta, int scalars_on_device,
                                        const void* x, void* y, void* workspace);

/* The long tail of cusparseSpMV's real-valued argument space (spmv_generic.cu; SURVEY.md 8(f)-3): 64-bit indices, fp32 A with
 * fp64 x / y / arithmetic, transposes of those and of Sliced-ELL, CSR without a workspace.  Plain plan-free kernels.
 *   off64 / col64 / idx64 : 0 = int32, 1 = int64 (CUSPARSE_INDEX_32I / _64I, cusparse.h:5002-5007); 32-bit offsets with 64-bit
 *                           columns are rejected (-1)
 *   a_dtype               : type of A's values; xy_dtype: type of x, y, alpha, beta and of the arithmetic (0 = fp32, 1 = fp64);
 *                           a_dtype <= xy_dtype
 *   transpose             : 0: y[rows] = alpha*A*x[cols] + beta*y;  1: y[cols] = alpha*A^T*x[rows] + beta*y (fp atomics)
 * COO: A^T is the same call with row_ind / col_ind and rows / cols swapped. */
B200SPMV_EXPORT int b200spmv_csr_generic_mv(void* stream, int off64, int col64, int a_dtype, int xy_dtype, int transpose,
                                            int64_t rows, int64_t cols, int64_t nnz, const void* row_offsets, const void* col_ind,
                                            const void* values, int64_t base, const void* alpha, const void* beta,
                                            int scalars_on_device, const void* x, void* y);
B200SPMV_EXPORT int b200spmv_coo_generic_mv(void* stream, int idx64, int a_dtype, int xy_dtype, int64_t rows, int64_t cols,
                                            int64_t nnz, const void* row_ind, const void* col_ind, const void* values, int64_t base,
                                            const void* alpha, const void* beta, int scalars_on_device, const void* x, void* y);
B200SPMV_EXPORT int b200spmv_sell_generic_mv(void* stream, int off64, int col64, int a_dtype, int xy_dtype, int transpose,
                                             int64_t rows, int64_t cols, int64_t slice_size, const void* slice_offsets,
                                             const void* col_ind, const void* values, int64_t base, const void* alpha,
                                             const void* beta, int scalars_on_device, const void* x, void* y);

/* Run-time switches (tests / tuning sweeps; never needed by a caller).  The environment variables of the same names
 * are read ONCE at first use; afterwards only this call changes them.  Not thread-safe against concurrent launches.
 *   B200SPMV_CSR_KERNEL = auto|tile|pipe|ws|rowwise|seg     B200SPMV_COO_KERNEL = auto|tile|seg
 *   B200SPMV_FLAT = auto|on|off   B200SPMV_FLAT_QUIET = <permille>
 *   B200SPMV_TILE_ORDER = scatter|linear   B200SPMV_PDL = 0|1   B200SPMV_SEG_DENSE = <nnz per row>   B200SPMV_SELL_GENERIC = 0|1
 *   B200SPMV_SHORT = auto|on|off
 *   B200SPMV_GENERIC = off|csr|all (what spmv_generic.cu serves instead of the closed library: nothing / CSR [default] / also
 *                      COO, Sliced-ELL and strided-batch SpMM, which have not had their first hardware run yet)
 * returns 0, or -1 for an unknown key / value. */
B200SPMV_EXPORT int  b200spmv_set_option(const char* key, const char* value);
/* Call counters of the cuSPARSE-symbol layer: SpMV calls that ran on our kernels, SpMV calls handed to the closed library
 * (unsupported combination, NULL / misaligned buffer, B200SPMV_FORWARD=1), CSR analyses run.  Tests assert
 * forwarded == 0 on the hot path. */
B200SPMV_EXPORT void b200spmv_get_stats(uint64_t* native_calls, uint64_t* forwarded_calls, uint64_t* analyze_calls);
B200SPMV_EXPORT void b200spmv_reset_stats(void);
/* Which path cusparseSpMV takes for a call of this shape (enum values of cusparse.h / library_types.h passed as int):
 * 0 = handed to the closed library, 1 = the specialised 32-bit-index single-type kernels, 2 = spmv_generic.cu.  Host logic only. */
B200SPMV_EXPORT int b200spmv_route(int format, int op, int alg, int off_type, int col_type, int a_vtype, int x_vtype, int y_vtype,
                                   int compute_type, int64_t rows, int64_t cols, int64_t nnz);
/* How many products cusparseSpMM would run on our kernel for these descriptors (cusparseSpMatDescr_t / cusparseDnMatDescr_t passed
 * as void*): 0 = the call goes to the closed library, 1 = an ordinary product, N = a strided batch.  Host logic only. */
B200SPMV_EXPORT int b200spmm_batch_count(const void* matA, const void* matB, const void* matC);
/* name of the main kernel the most recent CSR SpMV launched, e.g. "b200::csr_seg_kernel<double>" (bench.py's roofline.kernel) */
B200SPMV_EXPORT const char* b200spmv_last_csr_kernel(void);

B200SPMV_EXPORT const char* b200spmv_version(void);

#ifdef __cplusplus
}
#endif

/* ============================================================================================== *
 * Layer 1: the cuSPARSE symbols re-exported by the shim (prototypes == /usr/local/cuda/include/   *
 * cusparse.h of CUDA 12.9; the line numbers cite that header, the call sites cite the reference). *
 * Compile with -DB200SPMV_DECLARE_CUSPARSE (and cusparse.h on the include path) to see them.      *
 * ============================================================================================== */
#ifdef B200SPMV_DECLARE_CUSPARSE
#include <cusparse.h>
#ifdef __cplusplus
extern "C" {
#endif
/* cusparse.h:5208 -- spmv_csr_example.c:88-91, cg_example.c:387-395, bicgstab_example.c:465-484 */
B200SPMV_EXPORT cusparseStatus_t cusparseCreateCsr(cusparseSpMatDescr_t*, int64_t, int64_t, int64_t, void*, void*, void*,
                                                   cusparseIndexType_t, cusparseIndexType_t, cusparseIndexBase_t, cudaDataType);
/* cusparse.h:5221 -- cuSOLVERSp2cuDSS/csreigvsi2cuDSS_double.cpp:139-141 */
B200SPMV_EXPORT cusparseStatus_t cusparseCreateConstCsr(cusparseConstSpMatDescr_t*, int64_t, int64_t, int64_t, const void*,
                                                        const void*, const void*, cusparseIndexType_t, cusparseIndexType_t,
                                                        cusparseIndexBase_t, cudaDataType);
/* cusparse.h:5362 -- spmv_coo_example.c:86-89 */
B200SPMV_EXPORT cusparseStatus_t cusparseCreateCoo(cusparseSpMatDescr_t*, int64_t, int64_t, int64_t, void*, void*, void*,
                                                   cusparseIndexType_t, cusparseIndexBase_t, cudaDataType);
/* cusparse.h:5374 */
B200SPMV_EXPORT cusparseStatus_t cusparseCreateConstCoo(cusparseConstSpMatDescr_t*, int64_t, int64_t, int64_t, const void*,
                                                        const void*, const void*, cusparseIndexType_t, cusparseIndexBase_t,
                                                        cudaDataType);
/* cusparse.h:5470 -- spmv_sell_example.c:103-107 */
B200SPMV_EXPORT cusparseStatus_t cusparseCreateSlicedEll(cusparseSpMatDescr_t*, int64_t, int64_t, int64_t, int64_t, int64_t,
                                                         void*, void*, void*, cusparseIndexType_t, cusparseIndexType_t,
                                                         cusparseIndexBase_t, cudaDataType);
/* cusparse.h:5485 */
B200SPMV_EXPORT cusparseStatus_t cusparseCreateConstSlicedEll(cusparseConstSpMatDescr_t*, int64_t, int64_t, int64_t, int64_t,
                                                              int64_t, const void*, const void*, const void*,
                                                              cusparseIndexType_t, cusparseIndexType_t, cusparseIndexBase_t,
                                                              cudaDataType);
/* cusparse.h:5137 -- spmv_csr_example.c:115 */
B200SPMV_EXPORT cusparseStatus_t cusparseDestroySpMat(cusparseConstSpMatDescr_t);
/* cusparse.h:5312 / 5410 / 5156: keep the side table coherent when pointers are swapped */
B200SPMV_EXPORT cusparseStatus_t cusparseCsrSetPointers(cusparseSpMatDescr_t, void*, void*, void*);
B200SPMV_EXPORT cusparseStatus_t cusparseCooSetPointers(cusparseSpMatDescr_t, void*, void*, void*);
B200SPMV_EXPORT cusparseStatus_t cusparseSpMatSetValues(cusparseSpMatDescr_t, void*);
/* cusparse.h:5175 -- spmm_csr_batched_example.c:140 (the library has no getter for the strides: the shim records them) */
B200SPMV_EXPORT cusparseStatus_t cusparseCsrSetStridedBatch(cusparseSpMatDescr_t, int, int64_t, int64_t);
/* cusparse.h:5094 / 5100 / 5106 / 5129 -- spmv_csr_example.c:93-95,116-117, cg_example.c:371-378 */
B200SPMV_EXPORT cusparseStatus_t cusparseCreateDnVec(cusparseDnVecDescr_t*, int64_t, void*, cudaDataType);
B200SPMV_EXPORT cusparseStatus_t cusparseCreateConstDnVec(cusparseConstDnVecDescr_t*, int64_t, const void*, cudaDataType);
B200SPMV_EXPORT cusparseStatus_t cusparseDestroyDnVec(cusparseConstDnVecDescr_t);
B200SPMV_EXPORT cusparseStatus_t cusparseDnVecSetValues(cusparseDnVecDescr_t, void*);
/* cusparse.h:5691 -- spmv_csr_example.c:97-100, cg_example.c:409-412 */
B200SPMV_EXPORT cusparseStatus_t cusparseSpMV_bufferSize(cusparseHandle_t, cusparseOperation_t, const void*,
                                                         cusparseConstSpMatDescr_t, cusparseConstDnVecDescr_t, const void*,
                                                         cusparseDnVecDescr_t, cudaDataType, cusparseSpMVAlg_t, size_t*);
/* cusparse.h:5703 -- spmv_csr_example.c:104-107, csreigvsi2cuDSS_double.cpp:148-150 */
B200SPMV_EXPORT cusparseStatus_t cusparseSpMV_preprocess(cusparseHandle_t, cusparseOperation_t, const void*,
                                                         cusparseConstSpMatDescr_t, cusparseConstDnVecDescr_t, const void*,
                                                         cusparseDnVecDescr_t, cudaDataType, cusparseSpMVAlg_t, void*);
/* cusparse.h:5679 -- spmv_csr_example.c:110-112, cg_example.c:156,220,294,415,
 *                    bicgstab_example.c:190,262,315,358,504 */
B200SPMV_EXPORT cusparseStatus_t cusparseSpMV(cusparseHandle_t, cusparseOperation_t, const void*, cusparseConstSpMatDescr_t,
                                              cusparseConstDnVecDescr_t, const void*, cusparseDnVecDescr_t, cudaDataType,
                                              cusparseSpMVAlg_t, void*);
/* cusparse.h:5862-5898 -- spmm_csr_example.c:105-132, spmm_csr_batched_example.c:138-160 (dense-matrix descriptors stay with
 * the real library: the shim reads them through cusparseConstDnMatGet / cusparseDnMatGetStridedBatch, so cusparseCreateDnMat /
 * cusparseDnMatSetStridedBatch / cusparseDestroyDnMat need no re-export) */
B200SPMV_EXPORT cusparseStatus_t cusparseSpMM_bufferSize(cusparseHandle_t, cusparseOperation_t, cusparseOperation_t, const void*,
                                                         cusparseConstSpMatDescr_t, cusparseConstDnMatDescr_t, const void*,
                                                         cusparseDnMatDescr_t, cudaDataType, cusparseSpMMAlg_t, size_t*);
B200SPMV_EXPORT cusparseStatus_t cusparseSpMM_preprocess(cusparseHandle_t, cusparseOperation_t, cusparseOperation_t, const void*,
                                                         cusparseConstSpMatDescr_t, cusparseConstDnMatDescr_t, const void*,
                                                         cusparseDnMatDescr_t, cudaDataType, cusparseSpMMAlg_t, void*);
B200SPMV_EXPORT cusparseStatus_t cusparseSpMM(cusparseHandle_t, cusparseOperation_t, cusparseOperation_t, const void*,
                                              cusparseConstSpMatDescr_t, cusparseConstDnMatDescr_t, const void*,
                                              cusparseDnMatDescr_t, cudaDataType, cusparseSpMMAlg_t, void*);
#ifdef __cplusplus
}
#endif
#endif /* B200SPMV_DECLARE_CUSPARSE */

/* Shim behaviour switches (environment, read once at first use):
 *   B200SPMV_FORWARD=1   cusparseSpMV* forward to the real libcusparse (A/B oracle runs, same binary)
 *   B200SPMV_LOG=1       one line per call on stderr naming the path taken
 *   B200SPMV_CUSPARSE=/path/to/libcusparse.so.12   which real library to dlopen
 */
#endif /* B200SPMV_H_ */
