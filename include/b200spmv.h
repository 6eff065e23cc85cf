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

/* CSR in half precision (spmv_csr16.cu): y = alpha * A * x + beta * y, A rows x cols CSR.  Replaces cusparseSpMV for a CSR A with
 * fp16 / bf16 values and fp32 compute, opA = NON_TRANSPOSE.  Plan-free: needs no preprocess.
 *   a_type    : type of A's values and of x: 2 = fp16, 14 = bf16 (cudaDataType).
 *   y_type    : a_type or 0 = fp32.  alpha / beta (fp32, host or device) and the accumulation are fp32; the epilogue
 *               alpha * acc + beta * y is fp32 and rounds once to y_type.
 *   offsets   : rows + 1 int32 row offsets, columns: nnz int32 column indices, both with index base `base`.
 *   workspace : b200spmv_csr16_workspace_bytes() bytes, 16-byte aligned: two fp32 carry slots per chunk of
 *               b200spmv_csr16_params()'s chunk entries, so that a row crossing chunks is spread over their warps (split walk).  A
 *               NULL, misaligned or smaller buffer makes the warp of a row's first chunk add the row's later pieces itself (unsplit
 *               walk).
 * Bit-identity: the entries are cut into chunks at fixed positions; the sum of a row's piece inside a chunk depends only on that
 * piece's products (exact in fp32) and its position in the chunk, and a row adds its pieces in ascending chunk order.  So both walks,
 * repeated calls and graph replays give identical bits, on any grid or SM count.  Write-once: every y entry and every carry slot is
 * written exactly once, with no atomics; beta == 0 never reads y; an empty row gets beta * y; nothing past nnz is read, and x only
 * at stored columns.  No allocation, no host synchronisation (graph-capturable).  Sets b200spmv_last_csr_kernel(). */
B200SPMV_EXPORT int    b200spmv_csr16(void* stream, int a_type, int y_type, int64_t rows, int64_t cols, int64_t nnz, const void* offsets,
                                      const void* columns, const void* values, int32_t base, const void* alpha, const void* beta,
                                      int scalars_on_device, const void* x, void* y, void* workspace, size_t workspace_bytes);
/* 2 * ceil(nnz / chunk) * 4 bytes; 0 when rows or nnz is 0 */
B200SPMV_EXPORT size_t b200spmv_csr16_workspace_bytes(int64_t rows, int64_t nnz);
/* How b200spmv_csr16 streams these arrays: 2 = two entries per lane per load (64-bit columns, 32-bit value pairs: columns 8-byte
 * and values 4-byte aligned), 1 = scalar loads (a view misaligned by one element).  x and y are always read element by element. */
B200SPMV_EXPORT int    b200spmv_csr16_path(const void* columns, const void* values);
/* spmv_csr16's constants: entries per chunk (E), entries per run (a piece adds the sums of the runs it covers), warps per CTA */
B200SPMV_EXPORT void   b200spmv_csr16_params(int32_t* chunk, int32_t* run, int32_t* warps);

/* CSR in double complex (spmv_csr_z.cu): y = alpha * op(A) * x + beta * y, A rows x cols CSR.  Replaces cusparseSpMV for a CSR A
 * with CUDA_C_64F values, x, y and compute.
 *   op        : 0 = NON_TRANSPOSE (x has cols entries, y rows), 1 = TRANSPOSE, 2 = CONJUGATE_TRANSPOSE (x has rows entries, y cols).
 *   offsets   : rows + 1 int32 row offsets, columns: nnz int32 column indices, both with index base `base`.
 *   values, x, y : cuDoubleComplex, 16-byte aligned (any cuDoubleComplex array is; a misaligned y, or values / x when nnz > 0, is
 *               rejected with -1).
 *   alpha, beta : cuDoubleComplex, on the host or (scalars_on_device) on the device.
 *   workspace : op = 0 only: b200spmv_csr_z_workspace_bytes() bytes, 16-byte aligned: two cuDoubleComplex carry slots per chunk of
 *               b200spmv_csr_z_params()'s chunk entries (split walk).  A NULL, misaligned or smaller buffer gives the unsplit walk, with
 *               the same bits.  op = 1 / 2 use none.
 * Arithmetic (fixed with correctly rounded intrinsics, no contraction): a product is (fma(ar, br, -(ai * bi)), fma(ar, bi, ai * br));
 * the epilogue is (fma(al_r, acc_r, fma(-al_i, acc_i, t_r)), fma(al_r, acc_i, fma(al_i, acc_r, t_i))) with t = beta * y as a
 * product, t = 0 when beta == 0.
 * op = 0 is deterministic as b200spmv_csr16 is: chunks at fixed positions, each piece of a row summed in a fixed order, pieces in
 * ascending chunk order; both walks, repeated calls and graph replays give identical bits, no atomics; beta == 0 never reads y and an
 * empty row gets beta * y.  op = 1 / 2 scale y by beta, then add alpha * (v * x[r]) (conj(v) for op = 2) into y[c] with two fp64
 * atomic adds per entry: the order of the additions is not fixed.  No allocation, no host synchronisation (graph-capturable).  Sets
 * b200spmv_last_csr_kernel().  Returns 0, -1 for a rejected argument, or a cudaError_t. */
B200SPMV_EXPORT int    b200spmv_csr_z(void* stream, int op, int64_t rows, int64_t cols, int64_t nnz, const void* offsets, const void* columns,
                                      const void* values, int32_t base, const void* alpha, const void* beta, int scalars_on_device,
                                      const void* x, void* y, void* workspace, size_t workspace_bytes);
/* 2 * ceil(nnz / chunk) * 16 bytes; 0 when rows or nnz is 0 */
B200SPMV_EXPORT size_t b200spmv_csr_z_workspace_bytes(int64_t rows, int64_t nnz);
/* spmv_csr_z's constants: entries per chunk (E), entries per run (a piece adds the sums of the runs it covers), warps per CTA */
B200SPMV_EXPORT void   b200spmv_csr_z_params(int32_t* chunk, int32_t* run, int32_t* warps);

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

/* COO x dense (spmm_coo.cu): C = alpha * op(A) * B + beta * C, A rows x cols in COO (int32 row_ind / col_ind, index base `base`),
 * op(A) = A (transpose_a = 0) or A^T (1), B op(A).cols x n and C op(A).rows x n, each row- or column-major with leading dimension
 * ld* (elements).  Replaces cusparseSpMM for COO descriptors (cuSPARSE/spmm_coo/spmm_coo_example.c:110-122).
 *   batch     : 1..65535 products in one launch; product i uses row_ind / col_ind / values + i * a_stride, B + i * b_stride and
 *               C + i * c_stride (elements; 0 = shared by the batch; with batch > 1 the outputs must not overlap).
 *   workspace : b200spmm_coo_workspace_bytes() bytes, 16-byte aligned: per-batch "unsorted" flags (int32 at
 *               flag_offset + 4 * i of b200spmm_coo_params), the carry slots of the sorted path, and a row-major copy of a
 *               column-major B (n >= 4).
 * Row-sorted A with NON_TRANSPOSE runs deterministically without atomics (identical bits on every call); an unsorted A (any
 * descending pair of row indices, detected on the device), transpose_a = 1, or a NULL / misaligned / too small workspace runs on
 * the atomic path (B read in place when there is no workspace).  beta == 0 never reads C.  No allocation, no host synchronisation. */
B200SPMV_EXPORT size_t b200spmm_coo_workspace_bytes(int dtype, int transpose_a, int64_t rows, int64_t cols, int64_t n, int64_t nnz,
                                                    int b_row_major, int batch, int64_t b_stride);
B200SPMV_EXPORT int b200spmm_coo(void* stream, int dtype, int transpose_a, int64_t rows, int64_t cols, int64_t n, int64_t nnz,
                                 const void* row_ind, const void* col_ind, const void* values, int32_t base, const void* alpha,
                                 const void* beta, int scalars_on_device, const void* B, int64_t ldb, int b_row_major, void* C,
                                 int64_t ldc, int c_row_major, int batch, int64_t a_stride, int64_t b_stride, int64_t c_stride,
                                 void* workspace, size_t workspace_bytes);
/* the COO SpMM kernels' constants: consecutive non-zeros per warp chunk, columns of B / C per warp, and the byte offset of the
 * per-batch unsorted flags in the workspace (1 after a call = the atomic path ran for that batch) */
B200SPMV_EXPORT void b200spmm_coo_params(int32_t* chunk_nnz, int32_t* panel_cols, int64_t* flag_offset);

/* Blocked-ELL x dense (spmm_bell.cu): C = alpha * A * B + beta * C, A rows x cols in bs x bs blocks, B cols x n, C rows x n.
 * Replaces cusparseSpMM for Blocked-ELL descriptors (cuSPARSE/spmm_blockedell/spmm_blockedell_example.cpp).
 *   a_type    : 2 = fp16 (CUDA_R_16F) or 14 = bf16 (CUDA_R_16BF), the type of A's values and of B.
 *   c_type    : a_type or 0 = fp32 (CUDA_R_32F).  Products are accumulated in fp32; alpha / beta are fp32.
 *   col_ind   : (rows / bs) x (ell_cols / bs) int32 block columns, row-major, index base `base`; -1 marks an empty slot.
 *   values    : rows x ell_cols, row-major: row r holds its block-row's blocks side by side, bs values per block.  The values of an
 *               empty slot are never read, and neither are the rows of B that no block references.
 *   B, C      : row- or column-major with leading dimensions ldb / ldc (elements, at least the tight one).
 * rows, cols and ell_cols must be multiples of bs.  bs % 16 == 0 with 16-byte aligned values / B and ldb % 8 == 0 runs on tensor
 * cores (mma.sync, fp32 accumulators); everything else on a scalar kernel.  Each C entry is written once in a fixed order (no
 * atomics: identical bits on every call); beta == 0 never reads C.  No workspace, no allocation, no host synchronisation. */
B200SPMV_EXPORT int b200spmm_bell(void* stream, int a_type, int c_type, int64_t rows, int64_t cols, int64_t n, int64_t bs, int64_t ell_cols,
                                  const void* col_ind, const void* values, int32_t base, const void* alpha, const void* beta,
                                  int scalars_on_device, const void* B, int64_t ldb, int b_row_major, void* C, int64_t ldc,
                                  int c_row_major);
/* bell_mma_kernel's constants: columns of C per CTA, K slabs of 16 in flight, and the most rows of C a CTA owns (a CTA owns
 * 64, 32 or 16 rows of one block-row, the largest of these that divides bs). */
B200SPMV_EXPORT void b200spmm_bell_params(int32_t* n_tile, int32_t* stages, int32_t* max_rows_per_cta);

/* Sampled dense-dense product (sddmm_csr.cu): C = alpha * (op(A) * op(B)) o spy(C) + beta * C for a CSR C of m x n (int32
 * offsets / columns, `values` updated in place, once per entry, no atomics), op(A) m x k and op(B) k x n dense.  Replaces
 * cusparseSDDMM (cuSPARSE/sddmm_csr/sddmm_csr_example.c:114-134).  Any dense layout is passed as element strides:
 *   op(A)(i, k) = A[i * sai + k * sak],   op(B)(k, j) = B[k * sbk + j * sbj]   (strides >= 0).
 * batch >= 1 products run in one launch; matrix b of the batch uses offsets + b * off_stride, col_ind / values + b * colval_stride,
 * A + b * a_stride, B + b * b_stride (elements; 0 = shared by the batch; colval_stride >= nnz when batch > 1).
 * workspace: b200sddmm_csr_workspace_bytes() bytes, 16-byte aligned, where an operand that is not K-contiguous (its k stride is not
 * 1) is copied to a tight K-contiguous matrix on every call; a NULL, misaligned or smaller buffer makes the kernel read that operand
 * with strided loads instead.  beta == 0 never reads C's values.  K = 0 gives C = beta * C. */
B200SPMV_EXPORT size_t b200sddmm_csr_workspace_bytes(int dtype, int64_t m, int64_t n, int64_t k, int64_t sai, int64_t sak, int64_t sbk,
                                                     int64_t sbj, int batch, int64_t a_stride, int64_t b_stride);
B200SPMV_EXPORT int b200sddmm_csr(void* stream, int dtype, int64_t m, int64_t n, int64_t k, int64_t nnz, const void* row_offsets,
                                  const void* col_ind, void* values, int32_t base, const void* alpha, const void* beta,
                                  int scalars_on_device, const void* A, int64_t sai, int64_t sak, const void* B, int64_t sbk,
                                  int64_t sbj, int batch, int64_t off_stride, int64_t colval_stride, int64_t a_stride,
                                  int64_t b_stride, void* workspace, size_t workspace_bytes);
/* sddmm_csr_kernel's constants: consecutive non-zeros per warp, entries a lane group has in flight, the width of the vector loads of
 * the K-contiguous path, the widest lane group.  G lanes share one entry: G = the smallest power of two with G * V >= k, at most
 * max_group, where V = vec_bytes / sizeof(value) on the K-contiguous path (k a multiple of V, operands 16-byte aligned) and 1 on
 * the strided path; a warp steps through its chunk 32 / G * entries_per_group entries at a time. */
B200SPMV_EXPORT void b200sddmm_params(int32_t* warp_chunk, int32_t* entries_per_group, int32_t* vec_bytes, int32_t* max_group);

/* Sampled dense-dense product for a BSR C (sddmm_bsr.cu): C = alpha * (op(A) * op(B)) o spy(C) + beta * C, C m x n in square
 * bs x bs blocks (m and n multiples of bs), op(A) m x k and op(B) k x n dense.  Replaces cusparseSDDMM for BSR descriptors
 * (cuSPARSE/sddmm_bsr/sddmm_bsr_example.c).
 *   ab_type   : type of A and B: 0 = fp32, 1 = fp64 (cudaDataType CUDA_R_32F / _64F), 2 = fp16, 14 = bf16.
 *   c_type    : ab_type, or 0 = fp32 for 16-bit A and B.  alpha / beta and the accumulation are fp64 for fp64, fp32 otherwise.
 *   offsets   : m / bs + 1 int32 block offsets, columns: bnnz int32 block columns, both with index base `base`.
 *   values    : bnnz blocks of bs * bs values, each row-major (c_row_major = 1) or column-major inside the block.
 *   A, B      : op(A)(i, k) = A[i * sai + k * sak], op(B)(k, j) = B[k * sbk + j * sbj] (element strides >= 0, as b200sddmm_csr).
 * batch >= 1 products run in one launch; matrix b uses offsets + b * off_stride, columns + b * col_stride, values + b * val_stride,
 * A + b * a_stride, B + b * b_stride (elements; 0 = shared; val_stride >= bnnz * bs * bs when batch > 1).
 * 16-bit A and B with bs % 16 == 0 run on tensor cores (mma.sync, fp32 accumulators) when b200sddmm_bsr_path() says so; fp32 / fp64
 * and every other 16-bit call run on CUDA cores (FFMA / DFMA).  Each C entry is written once in a fixed k order (no atomics:
 * identical bits on every call), rounded once to C's type; beta == 0 never reads C; K = 0 gives C = beta * C.  Nothing is read
 * past K, in ld padding, or in rows / columns of op(A) / op(B) that no stored block references.  No workspace, no allocation, no
 * host synchronisation. */
B200SPMV_EXPORT int b200sddmm_bsr(void* stream, int ab_type, int c_type, int64_t m, int64_t n, int64_t k, int64_t bs, int64_t bnnz,
                                  const void* offsets, const void* columns, void* values, int32_t base, int c_row_major,
                                  const void* alpha, const void* beta, int scalars_on_device, const void* A, int64_t sai, int64_t sak,
                                  const void* B, int64_t sbk, int64_t sbj, int batch, int64_t off_stride, int64_t col_stride,
                                  int64_t val_stride, int64_t a_stride, int64_t b_stride);
/* 1 when b200sddmm_bsr runs these operands on tensor cores (16-bit, bs % 16 == 0, A and B 16-byte aligned, each operand contiguous
 * along K or along its other dimension with the other stride and the batch strides multiples of 8), 0 for the CUDA-core kernel. */
B200SPMV_EXPORT int b200sddmm_bsr_path(int ab_type, int64_t bs, const void* A, int64_t sai, int64_t sak, const void* B, int64_t sbk,
                                       int64_t sbj, int batch, int64_t a_stride, int64_t b_stride);
/* sddmm_bsr's constants: K of one tensor-path slab, slabs in flight, the widest block one tensor-path CTA owns whole (a wider block
 * is split into max_tile x max_tile tiles along its rows and columns, never along K), threads of a CUDA-core CTA. */
B200SPMV_EXPORT void b200sddmm_bsr_params(int32_t* k_slab, int32_t* stages, int32_t* max_tile, int32_t* fma_threads);

/* BSR x dense (spmm_bsr.cu): C = alpha * A * op(B) + beta * C, A m x k in square bs x bs blocks (m and k multiples of bs), op(B)
 * k x n and C m x n dense.  Replaces cusparseSpMM for BSR descriptors: the P . V of block-sparse attention.
 *   ab_type   : type of A's values and of B: 0 = fp32, 1 = fp64, 2 = fp16, 14 = bf16 (cudaDataType).
 *   c_type    : ab_type, or 0 = fp32 for 16-bit A and B.  alpha / beta and the accumulation are fp64 for fp64, fp32 otherwise.
 *   offsets   : m / bs + 1 int32 block offsets, columns: bnnz int32 block columns, both with index base `base`.
 *   values    : bnnz blocks of bs * bs values, each row-major (a_row_major = 1) or column-major inside the block.
 *   B         : op(B)(k, j) = B[k * sbk + j * sbj] (element strides >= 0, as b200sddmm_bsr).
 *   C         : row- or column-major with leading dimension ldc (elements).
 * batch >= 1 products run in one launch; matrix b uses offsets + b * off_stride, columns + b * col_stride, values + b * val_stride,
 * B + b * b_stride, C + b * c_stride (elements; 0 = shared, except C, whose matrices must not overlap).
 *   workspace : b200spmm_bsr_workspace_bytes() bytes, 16-byte aligned: carry slots that let a long block-row be split over several
 *               CTAs.  A NULL, misaligned or smaller buffer runs one CTA per block-row; both give identical bits.
 * 16-bit A and B with bs % 16 == 0 run on tensor cores (mma.sync, fp32 accumulators) when b200spmm_bsr_path() says so; fp32 / fp64
 * and every other call on CUDA cores (FFMA / DFMA).  Each C entry is written once in a fixed order (no atomics: identical bits on
 * every call); beta == 0 never reads C; block-rows that store nothing get beta * C.  Nothing is read past n, in ld padding, or in
 * rows of op(B) no stored block references.  No allocation, no host synchronisation. */
B200SPMV_EXPORT int b200spmm_bsr(void* stream, int ab_type, int c_type, int64_t m, int64_t k, int64_t n, int64_t bs, int64_t bnnz,
                                 const void* offsets, const void* columns, const void* values, int32_t base, int a_row_major,
                                 const void* alpha, const void* beta, int scalars_on_device, const void* B, int64_t sbk, int64_t sbj,
                                 void* C, int64_t ldc, int c_row_major, int batch, int64_t off_stride, int64_t col_stride,
                                 int64_t val_stride, int64_t b_stride, int64_t c_stride, void* workspace, size_t workspace_bytes);
B200SPMV_EXPORT size_t b200spmm_bsr_workspace_bytes(int ab_type, int64_t m, int64_t n, int64_t bs, int64_t bnnz, int batch);
/* 1 when b200spmm_bsr runs these operands on tensor cores (16-bit, bs % 16 == 0, row-major blocks, values and B 16-byte aligned,
 * op(B) contiguous along K or N with the other stride and the batch strides multiples of 8), 0 for the CUDA-core kernel. */
B200SPMV_EXPORT int b200spmm_bsr_path(int ab_type, int64_t bs, int a_row_major, const void* values, const void* B, int64_t sbk,
                                      int64_t sbj, int batch, int64_t val_stride, int64_t b_stride);
/* spmm_bsr's constants: K of one tensor-path slab, slabs per pipeline stage, stages in flight, the most rows of a block-row one
 * tensor-path CTA owns, and the piece length: a block-row is cut into pieces of ch = max(chunk_min, min(ceil(chunk_factor * bnnz /
 * (m / bs)), ceil(bnnz * batch * ceil(bs / 64) * ceil(n / 128) / target_ctas))) stored blocks, and with a workspace CTA c walks the
 * pieces that start in stored blocks [c * ch, (c + 1) * ch). */
B200SPMV_EXPORT void b200spmm_bsr_params(int32_t* k_slab, int32_t* slabs_per_stage, int32_t* stages, int32_t* max_rows_per_cta,
                                         int32_t* chunk_min, int32_t* chunk_factor, int32_t* target_ctas);

/* CSR x dense in half precision (spmm_csr16.cu): C = alpha * A * op(B) + beta * C, A m x k CSR, op(B) k x n and C m x n dense.
 * Replaces cusparseSpMM for a CSR A with fp16 / bf16 values and fp32 compute.
 *   ab_type   : type of A's values and of B: 2 = fp16, 14 = bf16 (cudaDataType).
 *   c_type    : ab_type or 0 = fp32.  alpha / beta (fp32, host or device) and the accumulation are fp32; the epilogue
 *               alpha * acc + beta * c is fp32 and rounds once to c_type.
 *   offsets   : m + 1 int32 row offsets, columns: nnz int32 column indices, both with index base `base`.
 *   B         : op(B)(k, j) = B[k * sbk + j * sbj] (element strides >= 0, as b200spmm_bsr).
 *   C         : row- or column-major with leading dimension ldc (elements).
 *   workspace : b200spmm_csr16_workspace_bytes() bytes, 16-byte aligned: the row-major copy of a K-contiguous op(B) (sbk == 1) and
 *               the carry slots that let a row longer than b200spmm_csr16_params()'s piece be split over several warps.  A NULL,
 *               misaligned or smaller buffer gathers op(B) in place and walks every row with one warp; both give identical bits.
 * fp32 FMAs on CUDA cores (no tensor cores: about one flop per gathered byte).  Each C entry is written once in a fixed order (no
 * atomics: identical bits on every call); beta == 0 never reads C; rows that store nothing get beta * C.  Nothing is read past n,
 * in ld padding, or in rows of op(B) no stored entry references.  No allocation, no host synchronisation. */
B200SPMV_EXPORT int b200spmm_csr16(void* stream, int ab_type, int c_type, int64_t m, int64_t k, int64_t n, int64_t nnz,
                                   const void* offsets, const void* columns, const void* values, int32_t base, const void* alpha,
                                   const void* beta, int scalars_on_device, const void* B, int64_t sbk, int64_t sbj, void* C, int64_t ldc,
                                   int c_row_major, void* workspace, size_t workspace_bytes);
B200SPMV_EXPORT size_t b200spmm_csr16_workspace_bytes(int64_t k, int64_t n, int64_t nnz, int64_t sbk, int64_t sbj);
/* How b200spmm_csr16 gathers these operands: the 16-bit elements per load, V (2, 4 or 8: one half2 / 64-bit / 128-bit load of a
 * lane's V columns, V = 1, 2, 4, 8 for n up to 32, 64, 128, more) or 1 (scalar loads: n <= 32, a misaligned view, a leading
 * dimension that is not a multiple of V, or op(B) not contiguous along n).  With a full workspace a K-contiguous op(B) is read
 * from its row-major copy: ask with (workspace, n, 1).  0 for bad arguments. */
B200SPMV_EXPORT int b200spmm_csr16_path(int64_t n, const void* B, int64_t sbk, int64_t sbj);
/* spmm_csr16's constants: the piece (a row is cut into pieces of at most this many entries at its start + multiples of it; a row
 * longer than one piece is split when there is a workspace), the entries of a row loaded per coalesced batch, the rows of a
 * row-tile CTA, warps per CTA, and the most columns of C one lane owns. */
B200SPMV_EXPORT void b200spmm_csr16_params(int32_t* piece, int32_t* lane_entries, int32_t* tile_rows, int32_t* warps,
                                           int32_t* max_cols_per_lane);

/* Transposed CSR x dense (spmm_csr_t.cu): C = alpha * op(A) * op(B) + beta * C with op(A) = A^T (= A^H: the types are real), A rows x
 * cols CSR with int32 offsets / columns (base 0 or 1), op(B) rows x n, C cols x n.  Replaces cusparseSpMM for a CSR A with opA =
 * TRANSPOSE / CONJUGATE_TRANSPOSE.  No atomics: a transposed plan (the CSC form of A's pattern) is built in the workspace, values are
 * gathered into it on every call, and the opA = N kernels run on A^T as a cols x rows CSR matrix (b200spmm_csr_ws for fp32 / fp64,
 * b200spmm_csr16 for fp16 / bf16).  The result is bit-identical to that opA = N call on the explicit transpose: deterministic.
 *   dtype / c_type : cudaDataType of A and B / of C: 0 / 0 (fp32), 1 / 1 (fp64), 2 or 14 / the same or 0 (fp16 or bf16, fp32 compute,
 *                    fp32 host or device scalars).
 *   B              : op(B)(k, j) = B[k * sbk + j * sbj].  fp32 / fp64 take op(B) row-major (sbj == 1) or column-major (sbk == 1).
 *   plan_valid     : nonzero when the workspace already holds the plan of this pattern (b200spmm_csr_t_plan or an earlier call with
 *                    the same offsets and columns), so only the values are gathered; 0 rebuilds the plan first.
 *   workspace      : b200spmm_csr_t_workspace_bytes() bytes, 16-byte aligned.
 * Returns -1 with nothing launched on a bad argument: unknown or mismatched types, a NULL, misaligned or short workspace, sizes past
 * the limits of the opA = N entry point, an fp32 / fp64 op(B) that is neither row- nor column-major.  No allocation, no host
 * synchronisation: graph-capturable. */
B200SPMV_EXPORT int b200spmm_csr_t(void* stream, int dtype, int c_type, int64_t rows, int64_t cols, int64_t n, int64_t nnz,
                                   const void* offsets, const void* columns, const void* values, int32_t base, const void* alpha,
                                   const void* beta, int scalars_on_device, const void* B, int64_t sbk, int64_t sbj, void* C, int64_t ldc,
                                   int c_row_major, int plan_valid, void* workspace, size_t workspace_bytes);
/* Builds the transposed plan of A's pattern in the workspace (at least offsets[4] of b200spmm_csr_t_layout bytes: the plan and the
 * sort scratch).  -1 on bad arguments, nothing launched. */
B200SPMV_EXPORT int b200spmm_csr_t_plan(void* stream, int64_t rows, int64_t cols, int64_t nnz, const void* offsets, const void* columns,
                                        int32_t base, void* workspace, size_t workspace_bytes);
/* The workspace of b200spmm_csr_t: total bytes (0 on bad arguments).  offsets (6 entries, or NULL) receives the byte offsets of
 * tOff (cols + 1 int32 CSC column pointers, base 0), tRow (nnz int32 rows, base 0, ascending within a column), perm (nnz int32 CSR
 * positions), the sort scratch, tVal (nnz values of A's type) and the opA = N kernel's own workspace.  Every part is 256-byte aligned;
 * the plan and the scratch depend on (cols, nnz) only. */
B200SPMV_EXPORT size_t b200spmm_csr_t_layout(int dtype, int64_t rows, int64_t cols, int64_t n, int64_t nnz, int64_t sbk, int64_t sbj,
                                             size_t* offsets);
B200SPMV_EXPORT size_t b200spmm_csr_t_workspace_bytes(int dtype, int64_t rows, int64_t cols, int64_t n, int64_t nnz, int64_t sbk,
                                                      int64_t sbj);

/* Format conversions (convert.cu), int32 indices, on the stable radix sort of the transposed plan: every result is a pure function
 * of the input, ties included.  Each returns -1 with nothing launched on a bad argument (negative or oversized sizes, a base other
 * than 0 / 1, a NULL or misaligned array the call needs, a NULL, misaligned or short workspace), else the CUDA launch status.  For
 * any index values, nothing is written outside the caller's outputs and workspace; out-of-range indices give an undefined result.
 * No allocation, no host synchronisation: graph-capturable.
 *
 * CSR -> CSC (cusparseCsr2cscEx2): A m x n CSR (base 0 or 1) to cscColPtr[n + 1] and cscRowInd[nnz] in the same base and, when
 * numeric is nonzero, cscVal[nnz] moved bit for bit, value_bytes 1, 2, 4, 8 or 16 wide.  Rows ascend within a column; duplicate
 * (row, col) entries keep their CSR order; columns need not be sorted within a row.  workspace: b200csr2csc_workspace_bytes()
 * bytes, 16-byte aligned (may be NULL when nnz = 0). */
B200SPMV_EXPORT int b200csr2csc(void* stream, int64_t m, int64_t n, int64_t nnz, const void* csr_val, const void* csr_row_ptr,
                                const void* csr_col_ind, void* csc_val, void* csc_col_ptr, void* csc_row_ind, int value_bytes, int numeric,
                                int32_t base, void* workspace, size_t workspace_bytes);
B200SPMV_EXPORT size_t b200csr2csc_workspace_bytes(int64_t m, int64_t n, int64_t nnz);
/* In-place COO sort (cusparseXcoosortByRow / ByColumn): rows and cols sorted lexicographically by (row, col) when by_row is nonzero,
 * else by (col, row); equal pairs keep their input order.  P gets the same permutation: P_out[i] = P_in[sigma(i)].  Keys are plain
 * ints in [0, m] / [0, n], so base 0 and base 1 both sort.  workspace: b200coosort_workspace_bytes() bytes, 16-byte aligned. */
B200SPMV_EXPORT int b200coosort(void* stream, int by_row, int64_t m, int64_t n, int64_t nnz, void* rows, void* cols, void* P,
                                void* workspace, size_t workspace_bytes);
B200SPMV_EXPORT size_t b200coosort_workspace_bytes(int64_t m, int64_t n, int64_t nnz);
/* cusparseXcoo2csr: csrRowPtr[m + 1] from the sorted cooRowInd[nnz], in the given base.  cusparseXcsr2coo: cooRowInd[nnz], the row
 * of each entry, from csrRowPtr[m + 1].  cusparseCreateIdentityPermutation: p[i] = i for i < n.  These three need no workspace. */
B200SPMV_EXPORT int b200coo2csr(void* stream, const void* coo_row_ind, int64_t nnz, int64_t m, void* csr_row_ptr, int32_t base);
B200SPMV_EXPORT int b200csr2coo(void* stream, const void* csr_row_ptr, int64_t nnz, int64_t m, void* coo_row_ind, int32_t base);
B200SPMV_EXPORT int b200identity_permutation(void* stream, int64_t n, void* p);

/* Sparse <-> dense conversion (dense_convert.cu), int32 indices, base 0 or 1.  The dense operand is rows x cols in order
 * 1 (CUSPARSE_ORDER_COL) or 2 (CUSPARSE_ORDER_ROW), the cusparseOrder_t values, with ld >= max(1, its contiguous dimension).  Values
 * move bit for bit by width (2, 4, 8 or 16 bytes).  No allocation, no host synchronisation, no floating-point atomics:
 * graph-capturable, and every result a pure function of the input.  Each returns -1 with nothing launched on bad sizes, base,
 * width, value type, order or ld, or on a NULL or misaligned pointer the call needs, else the CUDA launch status.
 *
 * Sparse -> dense (cusparseSparseToDense): every element of the m x n window of dense is written, zero where A has no entry;
 * nothing else is (not the ld padding).  Entries whose index lies outside the matrix are skipped.
 *   b200csr2dense   A m x n CSR (off[m + 1], ind = columns) or, with csc nonzero, CSC (off[n + 1], ind = rows), nnz entries
 *                   (ind / val may be NULL when nnz = 0); offsets are clamped to [0, nnz].  Duplicate entries within a row (CSC: a
 *                   column): the last in storage order wins.
 *   b200coo2dense   A as nnz (row, col) pairs; duplicate pairs leave one of their values.
 *   b200bell2dense  A Blocked-ELL: bs x bs blocks, colind[(m / bs) x (ell_cols / bs)] block columns (-1 or any index outside
 *                   the matrix: an empty slot, never read), val[m x ell_cols] row-major.  A block column named twice in a block
 *                   row: the last slot wins. */
B200SPMV_EXPORT int b200csr2dense(void* stream, int csc, int64_t m, int64_t n, int64_t nnz, const void* off, const void* ind, const void* val,
                                  int value_bytes, int32_t base, void* dense, int64_t ld, int order);
B200SPMV_EXPORT int b200coo2dense(void* stream, int64_t m, int64_t n, int64_t nnz, const void* rows, const void* cols, const void* val,
                                  int value_bytes, int32_t base, void* dense, int64_t ld, int order);
B200SPMV_EXPORT int b200bell2dense(void* stream, int64_t m, int64_t n, int64_t bs, int64_t ell_cols, const void* colind, const void* val,
                                   int value_bytes, int32_t base, void* dense, int64_t ld, int order);
/* Dense -> sparse (cusparseDenseToSparse_convert), after the closed library's analysis has written the offsets:
 *   b200dense2csr   CSR (or CSC, csc nonzero) columns (rows) and values of every non-zero of dense, in ascending order, line i
 *                   at off[i] - base onwards and never at or past off[i + 1] - base (both clamped to [0, nnz]): a line with more non-zeros than its range
 *                   keeps the first ones, one with fewer leaves the rest unwritten.  value_type: a cudaDataType among 16F, 16BF,
 *                   32F, 64F, C_32F and C_64F (complex fp16 / bf16 are refused: their predicate was not pinned); non-zero is
 *                   "v != 0" per part as the closed analysis counts it: denormals, Inf and NaN included, +-0 excluded -- and a
 *                   16-bit value whose magnitude bits exceed 0x7C00 excluded (that analysis reads fp16 and bf16 bits alike as
 *                   fp16: fp16 NaN; bf16 from about 2.7e36 up).
 *   b200dense2bell  val[m x ell_cols] of the Blocked-ELL matrix whose colind is given: each slot gets the dense bs x bs block it
 *                   names (zero past the matrix' edge); a slot of -1 (any index outside the matrix) gets zeros, as the closed
 *                   convert writes them. */
B200SPMV_EXPORT int b200dense2csr(void* stream, int csc, int64_t m, int64_t n, int64_t nnz, const void* dense, int64_t ld, int order,
                                  int value_type, const void* off, void* ind, void* val, int32_t base);
B200SPMV_EXPORT int b200dense2bell(void* stream, int64_t m, int64_t n, int64_t bs, int64_t ell_cols, const void* dense, int64_t ld,
                                   int order, int value_bytes, const void* colind, void* val, int32_t base);

/* Batched banded solves in the interleaved layout (batched_banded.cu; cusparse<t>gpsvInterleavedBatch / gtsvInterleavedBatch):
 * batch independent m x m systems A_j x_j = b_j, element i of system j at i * batch + j in every array.  vtype: CUDA_R_32F,
 * CUDA_R_64F, CUDA_C_32F or CUDA_C_64F (cudaDataType).  x holds the right-hand sides on entry and the solutions on return.  The
 * coefficient arrays are only read, and their out-of-band slots (ds[0..1], dl[0], du[m-1], dw[m-2..m-1] of every system) never.
 * workspace: the *_workspace_bytes() bytes, 16-byte aligned; it holds the triangular factor between the two sweeps.  One thread
 * per system, no atomics, no host synchronisation: graph-capturable, and each solution a pure function of its system.  -1 with
 * nothing launched on m or batch outside [1, INT32_MAX], an unknown vtype or algo, or a NULL or misaligned pointer; else the CUDA
 * launch status.  A singular factor gives Inf / NaN in x, as a division by zero does.
 *   b200gpsv_interleaved  pentadiagonal, row i = ds[i] x[i-2] + dl[i] x[i-1] + d[i] x[i] + du[i] x[i+1] + dw[i] x[i+2]: QR by Givens
 *                         rotations (complex: real c, complex s), R of upper bandwidth 4.
 *   b200gtsv_interleaved  tridiagonal, row i = dl[i] x[i-1] + d[i] x[i] + du[i] x[i+1]; algo 0: Thomas without pivoting (needs
 *                         non-zero pivots, e.g. diagonal dominance); 1: LU with partial pivoting; 2: QR by Givens rotations. */
B200SPMV_EXPORT int b200gpsv_interleaved(void* stream, int vtype, int64_t m, const void* ds, const void* dl, const void* d, const void* du,
                                         const void* dw, void* x, int64_t batch, void* workspace);
B200SPMV_EXPORT size_t b200gpsv_interleaved_workspace_bytes(int vtype, int64_t m, int64_t batch);
B200SPMV_EXPORT int b200gtsv_interleaved(void* stream, int vtype, int algo, int64_t m, const void* dl, const void* d, const void* du, void* x,
                                         int64_t batch, void* workspace);
B200SPMV_EXPORT size_t b200gtsv_interleaved_workspace_bytes(int vtype, int algo, int64_t m, int64_t batch);

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

/* The BLAS-1 part of an unpreconditioned BiCGStab iteration (cuSPARSE/bicgstab/bicgstab_example.c:212-351 with M = I), fused,
 * with every scalar AND every decision (convergence, breakdown) in device memory: no host synchronisation, CUDA-graph
 * capturable.  fp64; vectors 16-byte aligned; same walk, grid and deterministic reduction as b200cg_* (b200cg_params).
 * `workspace` = b200bicgstab_workspace_bytes() bytes, zeroed once by the caller; it also serves b200cg_dot (the arrival
 * counter sits at the same byte, max_ctas * 8, and every reduction leaves it at zero).
 * `state`: 16-byte aligned, b200bicgstab_state_layout(history_len) bytes: doubles at the B200BICGSTAB_* slot indices below,
 * then the int32 status, the int32 count of finished iterations, and history_len doubles of ||r|| (entry k after iteration
 * k, entry 0 = ||r0||; entries past history_len are not recorded).  The layout call reports the byte offsets.
 * One iteration, after r0 = b - A x0 and b200cg_dot(r0, r0 -> state[RHO_NEW]) then b200bicgstab_init:
 *   v = A p;  b200cg_dot(r0, v -> state[DENOM])
 *   b200bicgstab_update_s   alpha = rho_new / denom;  s = r - alpha v;  s2 = s . s;  rho <- rho_new
 *   t = A s;  b200bicgstab_dot2   ts = t . s,  tt = t . t
 *   b200bicgstab_update_xr  sqrt(s2) < threshold: x += alpha p, r = s, status CONVERGED_S;
 *                           else omega = ts / tt, x += alpha p + omega s, r = s - omega t;  then rho_new = r0 . r, r2 = r . r
 *   b200bicgstab_update_p   sqrt(r2) < threshold: status CONVERGED_R;
 *                           else beta = (rho_new / rho) (alpha / omega), p = r + beta (p - omega v)
 * A caller on several ranks all-reduces (sum) state[DENOM], then state[S2 .. TT] (contiguous), then state[RHO_NEW .. R2]
 * (contiguous) after the call that produced them; every decision is taken at kernel entry from those reduced values, so all
 * ranks stop at the same iteration.  A breakdown (denom = 0, tt = 0, omega = 0, rho_new = 0, or a non-finite scalar) sets its
 * status and updates nothing, so x never holds a NaN.  Once the status is not RUNNING every b200bicgstab_* iteration call
 * returns at entry: x, r, p and the state stay bit-identical (b200cg_dot still writes denom).  tol < 0: no convergence test.
 * Each call returns -1 with nothing launched on n < 0, a NULL or misaligned pointer (vectors may be NULL when n = 0), a
 * history_len outside [0, INT32_MAX] or a NaN tol; else the CUDA launch status. */
#define B200BICGSTAB_RHO        0      /* rho_{k-1}: r0 . r before this iteration */
#define B200BICGSTAB_ALPHA      1
#define B200BICGSTAB_OMEGA      2
#define B200BICGSTAB_DENOM      3      /* r0 . v */
#define B200BICGSTAB_S2         4      /* s . s   \                                        */
#define B200BICGSTAB_TS         5      /* t . s    | reduced (and all-reduced) together    */
#define B200BICGSTAB_TT         6      /* t . t   /                                        */
#define B200BICGSTAB_RHO_NEW    7      /* r0 . r  \ reduced together                       */
#define B200BICGSTAB_R2         8      /* r . r   /                                        */
#define B200BICGSTAB_THRESHOLD  9      /* tol * ||r0||, or -1 when there is no convergence test */
#define B200BICGSTAB_RUNNING             0
#define B200BICGSTAB_CONVERGED_S         1
#define B200BICGSTAB_CONVERGED_R         2
#define B200BICGSTAB_BREAKDOWN_DENOM     3
#define B200BICGSTAB_BREAKDOWN_TT        4
#define B200BICGSTAB_BREAKDOWN_OMEGA     5
#define B200BICGSTAB_BREAKDOWN_RHO       6
#define B200BICGSTAB_BREAKDOWN_NONFINITE 7
B200SPMV_EXPORT size_t b200bicgstab_workspace_bytes(void);
/* the state block's size in bytes for history_len history entries (0 when history_len is outside [0, INT32_MAX]); the byte
 * offsets of the status, the iteration counter and the history go to the non-NULL pointers */
B200SPMV_EXPORT size_t b200bicgstab_state_layout(int64_t history_len, int32_t* status_byte, int32_t* iter_byte, int32_t* history_byte);
/* r = p = r0;  rho = r2 = state[RHO_NEW];  threshold = tol * sqrt(rho);  counter 0;  history[0] = sqrt(rho);  status RUNNING,
 * CONVERGED_R when rho = 0 (x0 solves the system), BREAKDOWN_NONFINITE when rho is not finite */
B200SPMV_EXPORT int    b200bicgstab_init(void* stream, int64_t n, const double* r0, double* r, double* p, void* state,
                                         int64_t history_len, double tol);
B200SPMV_EXPORT int    b200bicgstab_update_s(void* stream, int64_t n, const double* r, const double* v, double* s, void* state,
                                             void* workspace);
B200SPMV_EXPORT int    b200bicgstab_dot2(void* stream, int64_t n, const double* t, const double* s, void* state, void* workspace);
B200SPMV_EXPORT int    b200bicgstab_update_xr(void* stream, int64_t n, double* x, double* r, const double* p, const double* s,
                                              const double* t, const double* r0, void* state, void* workspace);
B200SPMV_EXPORT int    b200bicgstab_update_p(void* stream, int64_t n, double* p, const double* r, const double* v, void* state);

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
 *   B200SPMV_ZCSR = auto|on (cusparseSpMV on a double-complex CSR A: auto [default] = b200spmv_csr_z only in the classes measured at
 *                      least at parity with the closed library (none today, DESIGN.md 3.21); on = every call in its class)
 *   B200SPMV_DENSE / B200SPMV_BANDED / B200SPMV_ILU0 / B200SPMV_SPGEMM = auto|on (the same choice for the conversions, the batched
 *                      banded solves, cusparse<t>csrilu02 / csric02 and cusparseSpGEMMreuse_compute)
 * returns 0, or -1 for an unknown key / value. */
B200SPMV_EXPORT int  b200spmv_set_option(const char* key, const char* value);
/* Call counters of the cuSPARSE-symbol layer: SpMV calls that ran on our kernels, SpMV calls handed to the closed library
 * (unsupported combination, NULL / misaligned buffer, B200SPMV_FORWARD=1), CSR analyses run.  Tests assert
 * forwarded == 0 on the hot path. */
B200SPMV_EXPORT void b200spmv_get_stats(uint64_t* native_calls, uint64_t* forwarded_calls, uint64_t* analyze_calls);
B200SPMV_EXPORT void b200spmv_reset_stats(void);
/* Which path cusparseSpMV takes for a call of this shape (enum values of cusparse.h / library_types.h passed as int):
 * 0 = handed to the closed library, 1 = the specialised 32-bit-index single-type kernels, 2 = spmv_generic.cu, 3 = b200spmv_csr16
 * (CSR, int32 indices, A and x fp16 or both bf16, y of A's type or fp32, fp32 compute, opA NON_TRANSPOSE, alg DEFAULT / CSR_ALG1 /
 * CSR_ALG2, in a class measured at least at parity with the closed library: DESIGN.md 3.19), 4 = b200spmv_csr_z (CSR, int32
 * indices, A, x, y and compute CUDA_C_64F, alg DEFAULT / CSR_ALG1 / CSR_ALG2, in a class measured at least at parity with the closed
 * library: DESIGN.md 3.21).  Host logic only. */
B200SPMV_EXPORT int b200spmv_route(int format, int op, int alg, int off_type, int col_type, int a_vtype, int x_vtype, int y_vtype,
                                   int compute_type, int64_t rows, int64_t cols, int64_t nnz);
/* The same decision over descriptors (cusparseSpMatDescr_t / cusparseDnVecDescr_t passed as void*), as cusparseSpMV_bufferSize /
 * _preprocess / cusparseSpMV take it: b200spmv_route's codes, 0 under B200SPMV_FORWARD=1 or for NULL descriptors, for descriptors of
 * any value type (complex ones included).  Host logic only. */
B200SPMV_EXPORT int b200spmv_csr16_route(const void* matA, const void* vecX, const void* vecY, int opA, int computeType, int alg);
/* How many products cusparseSpMM would run on our kernel for these descriptors (cusparseSpMatDescr_t / cusparseDnMatDescr_t passed
 * as void*): 0 = the call goes to the closed library, 1 = an ordinary product, N = a strided batch.  Host logic only. */
B200SPMV_EXPORT int b200spmm_batch_count(const void* matA, const void* matB, const void* matC);
/* Where cusparseSDDMM_bufferSize / _preprocess / cusparseSDDMM send a call with these descriptors (cusparseDnMatDescr_t A, B and
 * cusparseSpMatDescr_t C passed as void*, enum values as int): 0 = the closed library (64-bit indices, 16-bit / complex / mixed
 * types, a compute type other than the value type, non-CSR C, CONJUGATE_TRANSPOSE, an unsupported batch layout,
 * B200SPMV_FORWARD=1, and where the closed library measured faster: fp64, and fp32 with K > 32 when op(B) is K-contiguous),
 * 1 = one product on sddmm_csr_kernel, N = a strided batch of N.  Host logic only. */
B200SPMV_EXPORT int b200sddmm_route(const void* matA, const void* matB, const void* matC, int opA, int opB, int computeType);
/* Where cusparseSDDMM_bufferSize / _preprocess / cusparseSDDMM send a call with a BSR matC created through the shim: 0 = the closed
 * library, N >= 1 = N products on b200sddmm_bsr.  Native needs op NON_TRANSPOSE or TRANSPOSE, int32 indices, square blocks, A, B and
 * C of one real type (or 16-bit A and B with an fp32 C) with a compute type of fp32 (fp64 for fp64), a batch layout the closed
 * library accepts, no B200SPMV_FORWARD=1, and a class measured at least at parity with the closed library (DESIGN.md 3.16).  A BSR
 * descriptor created behind the shim's back is forwarded.  Host logic only. */
B200SPMV_EXPORT int b200sddmm_bsr_route(const void* matA, const void* matB, const void* matC, int opA, int opB, int computeType);
/* Where cusparseSpMM sends a call with a Blocked-ELL matA (descriptors passed as void*, enum values as int): 1 = b200spmm_bell,
 * 0 = the closed library.  Native needs NON_TRANSPOSE for both operands, alg DEFAULT or BLOCKED_ELL_ALG1, int32 block columns,
 * fp16 / bf16 A and B of one type, C of that type or fp32, compute type fp32, no strided batch, rows and cols multiples of the
 * block size, no B200SPMV_FORWARD=1, and a class measured at least at parity with the closed library (DESIGN.md 3.14).  A shape
 * mismatch between A, B and C stays native: the call rejects it.  Host logic only. */
B200SPMV_EXPORT int b200spmm_bell_route(const void* matA, const void* matB, const void* matC, int opA, int opB, int computeType, int alg);
/* Where cusparseSpMM_bufferSize / _preprocess / cusparseSpMM send a call with a COO matA (descriptors passed as void*, enum values as
 * int): 0 = the closed library, N >= 1 = N products on b200spmm_coo (a strided batch when N > 1).  Native needs opA NON_TRANSPOSE or
 * TRANSPOSE, opB NON_TRANSPOSE, alg DEFAULT / COO_ALG1 / COO_ALG3 / COO_ALG4 (COO_ALG2 promises bit-wise reproducibility for any entry
 * order and is forwarded), int32 indices, fp32 / fp64 A, B, C and compute of one type, a batch layout b200spmm_coo serves, no
 * B200SPMV_FORWARD=1, and a class measured at least at parity with the closed library (DESIGN.md 3.15).  A shape mismatch stays
 * native: the call rejects it.  Host logic only. */
B200SPMV_EXPORT int b200spmm_coo_route(const void* matA, const void* matB, const void* matC, int opA, int opB, int computeType, int alg);
/* Where cusparseSpMM_bufferSize / _preprocess / cusparseSpMM send a call with a BSR matA created through the shim (descriptors passed
 * as void*, enum values as int): 0 = the closed library, N >= 1 = N products on b200spmm_bsr (a strided batch when N > 1).  Native
 * needs opA NON_TRANSPOSE, opB NON_TRANSPOSE or TRANSPOSE, alg DEFAULT or BSR_ALG1, int32 indices, square blocks, A and B of one
 * type with C of that type (or 16-bit A and B with an fp32 C) and a compute type of fp32 (fp64 for fp64), a batch layout the closed
 * library accepts, no B200SPMV_FORWARD=1, and a class measured at least at parity with the closed library (DESIGN.md 3.17).  A shape
 * mismatch stays native: the call rejects it.  Host logic only. */
B200SPMV_EXPORT int b200spmm_bsr_route(const void* matA, const void* matB, const void* matC, int opA, int opB, int computeType, int alg);
/* Where cusparseSpMM_bufferSize / _preprocess / cusparseSpMM send a call with a CSR matA of fp16 / bf16 values: 1 = b200spmm_csr16,
 * 0 = the closed library.  Native needs opA NON_TRANSPOSE, opB NON_TRANSPOSE or TRANSPOSE, alg DEFAULT or CSR_ALG1 / 2 / 3, int32
 * indices, B of A's type, C of A's type or fp32, compute type fp32, no strided batch, no B200SPMV_FORWARD=1, and a class measured at
 * least at parity with the closed library (DESIGN.md 3.18).  A shape mismatch stays native: the call rejects it.  Host logic only. */
B200SPMV_EXPORT int b200spmm_csr16_route(const void* matA, const void* matB, const void* matC, int opA, int opB, int computeType, int alg);
/* Where cusparseSpMM sends a call with a CSR matA and opA TRANSPOSE / CONJUGATE_TRANSPOSE, given the call's externalBuffer: 1 =
 * b200spmm_csr_t, 0 = the closed library.  Native needs opA TRANSPOSE (the closed library refuses CONJUGATE_TRANSPOSE for these real
 * types: such calls keep its verdict), alg DEFAULT or CSR_ALG1, int32 indices, no strided batch, a non-NULL buffer,
 * no B200SPMV_FORWARD=1, opB NON_TRANSPOSE (opB = T was not measured); fp32 / fp64 with A, B, C and compute of one type, or fp16 /
 * bf16 with B of A's type, C of A's type or fp32 and compute fp32; and a class measured at least at parity with the closed library
 * (DESIGN.md 3.22).  Host logic only. */
B200SPMV_EXPORT int b200spmm_csr_t_route(const void* matA, const void* matB, const void* matC, int opA, int opB, int computeType, int alg,
                                         void* buffer);
/* Whether the shim trusts `buffer` to hold matA's plan of a kind: 0 = the CSR SpMV plan (cusparseSpMV_preprocess), 1 = the
 * transposed SpMM plan (cusparseSpMM_preprocess).  A buffer holds the plan of its latest preprocess only, and each kind trusts only
 * its own; cusparseCsrSetPointers, a new bufferSize query of that operation and cusparseDestroySpMat drop the trust.  Host logic only. */
B200SPMV_EXPORT int b200spmv_plan_trusted(const void* matA, void* buffer, int kind);
/* Where the shim sends a conversion call: 1 = the native entry point above, 0 = the closed library.  op: B200CONV_CSR2CSC (arg:
 * value bytes, 0 for CUSPARSE_ACTION_SYMBOLIC), B200CONV_COOSORT_ROW / _COL, B200CONV_COO2CSR, B200CONV_CSR2COO, B200CONV_IDENTITY
 * (arg unused); alg: cusparseCsr2CscAlg_t (csr2csc only); buffer: the call's buffer (csr2csc with nnz > 0 and coosort only).
 * Native needs CUSPARSE_CSR2CSC_ALG1, a non-NULL 16-byte aligned buffer where one is used, sizes within the sort's limits, no
 * B200SPMV_FORWARD=1, and a class measured at least at parity with the closed library (DESIGN.md 3.23).  Host logic only. */
#define B200CONV_CSR2CSC 0
#define B200CONV_COOSORT_ROW 1
#define B200CONV_COOSORT_COL 2
#define B200CONV_COO2CSR 3
#define B200CONV_CSR2COO 4
#define B200CONV_IDENTITY 5
B200SPMV_EXPORT int b200conv_route(int op, int64_t m, int64_t n, int64_t nnz, int arg, int alg, const void* buffer);
/* Where the shim sends cusparseSparseToDense (direction B200DENSE_S2D) or cusparseDenseToSparse_convert (B200DENSE_D2S): 1 = the
 * native entry point above, 0 = the closed library.  format: cusparseFormat_t of the sparse side; order: cusparseOrder_t of the
 * dense side; vtype: cudaDataType; off_type / col_type: cusparseIndexType_t; batch: the larger strided-batch count of the two
 * descriptors; alg: the call's algorithm; bs: the Blocked-ELL block size (ignored for other formats).  Forwarded:
 * B200SPMV_FORWARD=1, 64-bit indices, a base other than 0 / 1, integer, complex fp16 / bf16 or unknown value types for dense ->
 * CSR / CSC, dense -> COO, strided batches, an alg other than DEFAULT, and every class not measured at least at parity with the
 * closed library (DESIGN.md 3.24; today only dense -> Blocked-ELL, row-major, bs 16, fp16 / fp32, 8192 to 16384 rows and columns
 * is native).  B200SPMV_DENSE=on makes every call this admits native.  Host logic only. */
#define B200DENSE_S2D 0
#define B200DENSE_D2S 1
B200SPMV_EXPORT int b200dense_route(int direction, int format, int order, int vtype, int off_type, int col_type, int base, int64_t rows,
                                    int64_t cols, int64_t nnz, int batch, int alg, int64_t bs);
/* Where the shim sends cusparse<t>gpsvInterleavedBatch (op B200BAND_GPSV, algo 0) or cusparse<t>gtsvInterleavedBatch (op
 * B200BAND_GTSV, algo 0 / 1 / 2): 1 = b200gpsv_interleaved / b200gtsv_interleaved, 0 = the closed library.  vtype: cudaDataType;
 * buffer: the call's pBuffer.  Forwarded: B200SPMV_FORWARD=1, an algo outside that set, m < 3 or batch < 1 (the closed library
 * gives its own verdict on those), a NULL or misaligned buffer, and every class not measured at least at parity with the closed
 * library (DESIGN.md 3.25).  B200SPMV_BANDED=on makes every call this admits native.  Host logic only. */
#define B200BAND_GPSV 0
#define B200BAND_GTSV 1
B200SPMV_EXPORT int b200banded_route(int op, int vtype, int algo, int64_t m, int64_t batch, const void* buffer);
/* ---------------------------------------------------------------------------------------------- *
 * Sparse triangular solve with many right-hand sides (cusparseSpSM; cuSPARSE/spsm_csr):           *
 *   C = alpha op(T)^-1 op(B), T the selected triangle of the rows x rows CSR matrix A (int32       *
 *   offsets and columns, index base 0 or 1).  A may store both triangles: entries outside the      *
 *   selected one are ignored, and with unit = 1 so is the stored diagonal.  lower / unit /         *
 *   transpose as in b200spsv.h; dtype 0 = fp32, 1 = fp64 (values, B, C, alpha, arithmetic).        *
 *   return: 0, -1 on invalid arguments (checked before any CUDA call), else the cudaError_t.      *
 * ---------------------------------------------------------------------------------------------- */
/* Bytes of the workspace _analysis builds the plan in; pass it to every _solve of that plan (it also holds the solve-state
 * words, so two solves of one plan must not overlap). */
B200SPMV_EXPORT size_t b200spsm_csr_workspace_bytes(int64_t rows, int64_t nnz, int transpose);
/* Byte offsets of the plan's arrays (each 256-byte aligned): SpSV's plan (b200spsv.h: state words, flags, t_off, diag,
 * t_col, t_vidx) and order[rows], the rows in level order (by level, then by position in the solve direction); the scratch
 * comes last and the solve reads nothing from it.  offsets[B200SPSM_TOTAL] == b200spsm_csr_workspace_bytes(...).  Returns -1 for
 * negative sizes. */
enum { B200SPSM_STATE = 0, B200SPSM_FLAGS, B200SPSM_T_OFF, B200SPSM_DIAG, B200SPSM_T_COL, B200SPSM_T_VIDX, B200SPSM_ORDER, B200SPSM_SCRATCH,
       B200SPSM_TOTAL, B200SPSM_LAYOUT_N };
B200SPMV_EXPORT int b200spsm_csr_layout(int64_t rows, int64_t nnz, int transpose, size_t* offsets /* [B200SPSM_LAYOUT_N] */);
/* Builds the plan and the level order (integer work; values are not read) and clears the state words.  Synchronises the
 * stream: the levels are computed on the host from the plan read back.  missing_diag (unit = 0: rows without a stored
 * diagonal) and levels (the number of dependency levels) are written when not NULL. */
B200SPMV_EXPORT int b200spsm_csr_analysis(void* stream, int64_t rows, int64_t nnz, const void* row_offsets, const void* col_ind,
                                          int32_t base, int lower, int unit, int transpose, void* workspace, int64_t* missing_diag,
                                          int64_t* levels);
/* C = alpha op(T)^-1 op(B) with the plan in workspace, for 0 <= nrhs <= B200SPSM_MAX_NRHS right-hand sides: op(B)(i, j) = B[i * sbi + j * sbk] and
 * C(i, j) = C[i * sci + j * scj] (any layout, transpose and leading dimension).  values are read now; diag (rows values, or
 * NULL) replaces the stored diagonal.  alpha is a host pointer, or a device pointer read in the kernel (alpha_on_device = 1).
 * B may be C.  Two launches, no allocation, no host synchronisation: CUDA-graph capturable.  Each result's bits depend on
 * the plan and b200spsm_csr_tile(nrhs, scj == 1) only. */
#define B200SPSM_MAX_NRHS (INT32_MAX - 32)      /* the kernel steps tiles of up to 32 columns in int */
B200SPMV_EXPORT int b200spsm_csr_solve(void* stream, int dtype, int64_t rows, int64_t nnz, int unit, const void* values, const void* diag,
                                       const void* alpha, int alpha_on_device, int64_t nrhs, const void* B, int64_t sbi, int64_t sbk,
                                       void* C, int64_t sci, int64_t scj, void* workspace);
/* Right-hand sides per tile of the solve kernel: lanes over min(32, nrhs) columns of a C with unit column stride (row-major),
 * over (entry group, column) with at most 8 columns otherwise (DESIGN.md 3.20).  A power of two.  Pure. */
B200SPMV_EXPORT int b200spsm_csr_tile(int64_t nrhs, int c_row_major);
/* Threads per CTA of the solve kernel and the budget (ns of %globaltimer) of any one wait, as b200spsv_csr_params. */
B200SPMV_EXPORT void b200spsm_csr_params(int32_t* threads_per_cta, uint64_t* spin_budget_ns);
/* Where cusparseSpSM sends a call of this shape (enum values as int): 0 = the closed library (outside the scope above: not CSR,
 * 64-bit indices, types other than fp32 / fp64 of one type, CONJUGATE_TRANSPOSE, an alg other than DEFAULT, non-square A,
 * batch > 1), 1 = within that scope but not in a class measured at least at parity with the closed library (forwarded),
 * 2 = b200spsm_csr_solve (analysis may still forward a NON_UNIT matrix with a row that stores no diagonal).  No class is
 * measured native today, so every call in scope answers 1 (DESIGN.md 3.20).  Pure host logic. */
B200SPMV_EXPORT int b200spsm_route(int format, int opA, int opB, int alg, int off_type, int col_type, int a_vtype, int b_vtype, int c_vtype,
                                   int compute_type, int fill, int diag, int64_t rows, int64_t cols, int64_t nnz, int64_t nrhs,
                                   int c_row_major, int batch);
/* Since the last reset: SpSM solves run natively / SpSM calls handed to the closed library / native analyses. */
B200SPMV_EXPORT void b200spsm_get_stats(uint64_t* native_calls, uint64_t* forwarded_calls, uint64_t* analysis_calls);
B200SPMV_EXPORT void b200spsm_reset_stats(void);
/* ---------------------------------------------------------------------------------------------- *
 * Incomplete LU and Cholesky factorization without fill-in (cusparse<t>csrilu02 / csric02;       *
 * cuSPARSE/bicgstab, cuSPARSE/cg), ilu0_csr.cu:                                                  *
 *   the rows x rows CSR matrix A (int32 offsets and columns, index base 0 or 1, columns strictly  *
 *   ascending in every row) is overwritten in place by its factor.  A row without a stored        *
 *   diagonal is a structural zero: it is left as stored, and nothing is read from it.             *
 *   kind B200ILU0_LU: row i becomes L (unit, strictly lower) and U (upper with the diagonal).      *
 *   kind B200ILU0_IC: the lower triangle with the diagonal becomes L (A ~ L L^T); entries with     *
 *   column > row are never read or written.  dtype 0 = fp32, 1 = fp64.  Every operation is one    *
 *   correctly rounded mul / sub / div / sqrt, each entry a left fold in ascending column order    *
 *   (DESIGN.md 3.26): the bits are the plain sequential algorithm's, whatever the schedule.        *
 *   return: 0, -1 on invalid arguments (checked before any CUDA call), else the cudaError_t.      *
 * ---------------------------------------------------------------------------------------------- */
#define B200ILU0_LU 0
#define B200ILU0_IC 1
#define B200ILU0_BAD_PATTERN (-2)       /* analysis: a row with unsorted, duplicate or out-of-range columns, or offsets that decrease
                                           or leave [base, nnz + base] */
#define B200ILU0_NO_COOPERATIVE (-3)    /* analysis: the current device cannot launch cooperative kernels */
/* Bytes of the workspace analysis builds the schedule in; pass it to every factorization and zero-pivot query of that pattern. */
B200SPMV_EXPORT size_t b200ilu0_workspace_bytes(int64_t rows, int64_t nnz);
/* Byte offsets of the workspace's arrays, each 256-byte aligned: the state words (uint32: [4] levels, [5] zero-pivot row,
 * [6] rows with a bad pattern, [7] first row without a stored diagonal; INT32_MAX for "none"), diag[rows] (position of each
 * row's diagonal), order[rows] (rows by level, ascending within a level), level_start[rows + 1], then what only analysis uses:
 * SpSV's strictly-lower plan t_off / t_col / t_vidx, the offsets clamped to [base, nnz + base] and scratch.
 * offsets[B200ILU0_TOTAL] == b200ilu0_workspace_bytes(...).
 * Returns -1 for negative sizes. */
enum { B200ILU0_STATE = 0, B200ILU0_DIAG, B200ILU0_ORDER, B200ILU0_LEVEL_START, B200ILU0_T_OFF, B200ILU0_T_COL, B200ILU0_T_VIDX,
       B200ILU0_CHECKED_OFF, B200ILU0_SCRATCH, B200ILU0_TOTAL, B200ILU0_LAYOUT_N };
B200SPMV_EXPORT int b200ilu0_layout(int64_t rows, int64_t nnz, size_t* offsets /* [B200ILU0_LAYOUT_N] */);
/* Checks the pattern, finds each row's diagonal and the level schedule of the strictly-lower dependency graph (integer work;
 * values are not read).  The offsets are checked and clamped first, so no kernel indexes col_ind outside [0, nnz).  Synchronises
 * the stream once: the levels are computed on the host.  structural_zero receives the first
 * row without a stored diagonal, or -1; levels the number of levels.  Returns B200ILU0_BAD_PATTERN or B200ILU0_NO_COOPERATIVE
 * (nothing else in the workspace is then valid) as above. */
B200SPMV_EXPORT int b200ilu0_analysis(void* stream, int64_t rows, int64_t nnz, const void* row_offsets, const void* col_ind, int32_t base,
                                      void* workspace, int64_t* structural_zero, int64_t* levels);
/* Factorizes values in place on the schedule analysis built: one cooperative launch, warps take the rows of a level by static
 * striding, a grid-wide barrier between levels.  LU: with boost = 1, a pivot with |a_ii| <= *tol becomes *boost_val after its
 * row's updates.  tol (one double) and boost_val (one value of dtype) are host pointers, or device pointers read by the kernel
 * (on_device = 1); unused when boost = 0.  The zero-pivot word receives the smallest row whose pivot is zero (LU, after the
 * boost) or not positive (IC, before its square root), or the structural zero analysis found when that is smaller.  Rows without
 * a stored diagonal are left as stored, and a step whose row k has none is skipped: the factor is then defined, not meaningful.
 * No allocation, no host synchronisation. */
B200SPMV_EXPORT int b200ilu0_factor(void* stream, int kind, int dtype, int64_t rows, int64_t nnz, const void* row_offsets,
                                    const void* col_ind, int32_t base, void* values, int boost, const void* tol, const void* boost_val,
                                    int on_device, void* workspace);
/* The smallest row with a structural zero (analysis) or a zero pivot (the latest factorization), -1 for none, as
 * cusparseXcsrilu02_zeroPivot reports it: into the host int32 at position (on_device = 0), or by a kernel into the device int32 at
 * position (on_device = 1).  Synchronises the stream either way, as the closed call does, and writes the row to the host int64 at
 * row when not NULL. */
B200SPMV_EXPORT int b200ilu0_zero_pivot(void* stream, const void* workspace, void* position, int on_device, int64_t* row);
/* Threads per CTA of the factorization kernel and the CTAs per SM it launches at most. */
B200SPMV_EXPORT void b200ilu0_params(int32_t* threads_per_cta, int32_t* ctas_per_sm);
/* Where the shim's cusparse<t>csrilu02 / csric02 analysis sends a pattern (kind B200ILU0_LU / _IC, vtype: cudaDataType,
 * levels: b200ilu0_analysis' count): 1 = b200ilu0_factor, 0 = the closed library.  levels = 0 asks before analysis: 1 when some
 * level count could be native.  The shim asks that first, and where the answer is 0 (every call in the default mode today) its
 * bufferSize and analysis are the closed library's alone, with no native work.  Forwarded: B200SPMV_FORWARD=1, types other than
 * CUDA_R_32F / CUDA_R_64F, sizes outside int32, and every class not measured at least at parity with the closed library
 * (DESIGN.md 3.26).  B200SPMV_ILU0=on makes every call this admits native.  Host logic only. */
B200SPMV_EXPORT int b200ilu0_route(int kind, int vtype, int64_t rows, int64_t nnz, int64_t levels);
/* ---------------------------------------------------------------------------------------------- *
 * Sparse x sparse, numeric phase with structure reuse (cusparseSpGEMMreuse_compute;               *
 * cuSPARSE/spgemm_reuse), spgemm_csr.cu:                                                          *
 *   C = alpha A B + beta C on C's stored pattern, A rows x krows, B krows x cols, C rows x cols,  *
 *   all CSR with int32 offsets and columns, each with its own index base (0 or 1).  C's columns   *
 *   must be strictly ascending in every row; A's and B's need not be sorted, but a B row holds a  *
 *   column once.  dtype 0 = fp32, 1 = fp64 (values, alpha, beta, arithmetic).  Every C(i, j) is   *
 *   acc = fadd(acc, fmul(a_ik, b_kj)) from acc = +0 over A row i in stored order, then            *
 *   fadd(fmul(alpha, acc), fmul(beta, c_ij)), each correctly rounded (no FMA); at beta = 0 C is   *
 *   not read and the result is fmul(alpha, acc) (DESIGN.md 3.28).  The bits depend on nothing     *
 *   else.  A product whose column C's row does not store is skipped and counted in the plan.      *
 *   return: 0, -1 on invalid arguments (checked before any CUDA call), else the cudaError_t.      *
 * ---------------------------------------------------------------------------------------------- */
#define B200SPGEMM_BAD_PATTERN (-2)     /* plan: offsets outside [0, nnz] or decreasing, C columns not strictly ascending or outside
                                           [0, cols), A columns outside [0, krows), or a B row A names with bad offsets */
/* Bytes of the plan: a 256-byte header (64-bit words: [0] the bad-pattern bits, [1] products compute skipped because C's row does
 * not store their column, summed over every compute since the plan, [2] the compute kernel's pass queue, [3] the number of passes),
 * then each row's pass count and bin and the pass list.  A closed form of the sizes (nnz_a and nnz_b do not enter it today). */
B200SPMV_EXPORT size_t b200spgemm_plan_size(int64_t rows, int64_t nnz_a, int64_t nnz_b, int64_t nnz_c);
/* The C columns one warp stages in shared memory (a C row longer than this is cut into windows, each re-walking A's row), the
 * warps per CTA, and the three products-per-row edges of the four bins, heaviest first: bin b holds the rows with at least
 * bin_edges[b] products (bin 3: the rest).  Pure. */
B200SPMV_EXPORT void b200spgemm_params(int32_t* window, int32_t* warps_per_cta, int64_t* bin_edges /* [3] */);
/* Builds the plan from the three patterns (values are not read): checks them on the device, counts each C row's products
 * (int64), bins the rows and lists their windows heaviest bin first.  Synchronises the stream once, to read back the verdict:
 * B200SPGEMM_BAD_PATTERN (and the bits in *bad) when a pattern fails, else 0 with the pass count in *passes.  Nothing outside the
 * checked ranges is read. */
B200SPMV_EXPORT int b200spgemm_plan(void* stream, int64_t rows, int64_t krows, int64_t cols, int64_t nnz_a, int64_t nnz_b, int64_t nnz_c,
                                    const void* a_off, const void* a_col, int32_t a_base, const void* b_off, int32_t b_base,
                                    const void* c_off, const void* c_col, int32_t c_base, void* plan, size_t plan_bytes, int64_t* passes,
                                    uint64_t* bad);
/* C's values from the plan b200spgemm_plan built for these patterns (it must have returned 0).  alpha and beta are host pointers,
 * or device pointers read by the kernel (scalars_on_device = 1).  One memset and one launch: no allocation, no host
 * synchronisation, CUDA-graph capturable; two computes on one plan must not overlap. */
B200SPMV_EXPORT int b200spgemm_compute(void* stream, int dtype, int64_t rows, int64_t nnz_c, const void* a_off, const void* a_col,
                                       const void* a_val, int32_t a_base, const void* b_off, const void* b_col, const void* b_val,
                                       int32_t b_base, const void* c_off, const void* c_col, void* c_val, int32_t c_base,
                                       const void* alpha, const void* beta, int scalars_on_device, void* plan);
/* Where the shim sends cusparseSpGEMMreuse_copy's plan and cusparseSpGEMMreuse_compute (enum values as int; idx_*: the operand's
 * cusparseIndexType_t when its offsets and columns share it, else -1): 1 = b200spgemm_compute, 0 = the closed library.  Native
 * needs opA = opB = NON_TRANSPOSE, alg DEFAULT / CSR_ALG_DETERMINITIC / CSR_ALG_NONDETERMINITIC, three CSR operands with int32
 * indices and bases 0 / 1, A, B, C and the compute type all CUDA_R_32F or all CUDA_R_64F, every size below 2^31 - 1, no
 * B200SPMV_FORWARD=1, and a class measured at least at parity with the closed library (DESIGN.md 3.28: none today).
 * B200SPMV_SPGEMM=on makes every call this admits native.  Host logic only. */
B200SPMV_EXPORT int b200spgemm_route(int opA, int opB, int alg, int compute_type, int format_a, int format_b, int format_c, int vtype_a,
                                     int vtype_b, int vtype_c, int idx_a, int idx_b, int idx_c, int base_a, int base_b, int base_c,
                                     int64_t rows, int64_t krows, int64_t cols, int64_t nnz_a, int64_t nnz_b, int64_t nnz_c);
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
/* cusparse.h:5170 -- spmm_coo_batched_example.c:137 (one stride for the row, column and value arrays; recorded by the shim) */
B200SPMV_EXPORT cusparseStatus_t cusparseCooSetStridedBatch(cusparseSpMatDescr_t, int, int64_t);
/* cusparse.h:5327 / 5343 / 5181 -- sddmm_bsr_example.c (the library has no BSR getter: the shim records block size, block order
 * and the three batch strides) */
B200SPMV_EXPORT cusparseStatus_t cusparseCreateBsr(cusparseSpMatDescr_t*, int64_t, int64_t, int64_t, int64_t, int64_t, void*, void*,
                                                   void*, cusparseIndexType_t, cusparseIndexType_t, cusparseIndexBase_t, cudaDataType,
                                                   cusparseOrder_t);
B200SPMV_EXPORT cusparseStatus_t cusparseCreateConstBsr(cusparseConstSpMatDescr_t*, int64_t, int64_t, int64_t, int64_t, int64_t,
                                                        const void*, const void*, const void*, cusparseIndexType_t,
                                                        cusparseIndexType_t, cusparseIndexBase_t, cudaDataType, cusparseOrder_t);
B200SPMV_EXPORT cusparseStatus_t cusparseBsrSetStridedBatch(cusparseSpMatDescr_t, int, int64_t, int64_t, int64_t);
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
/* cusparse.h:6052-6088 -- sddmm_csr_example.c:114-134, sddmm_csr_batched_example.c:146-166 */
B200SPMV_EXPORT cusparseStatus_t cusparseSDDMM_bufferSize(cusparseHandle_t, cusparseOperation_t, cusparseOperation_t, const void*,
                                                          cusparseConstDnMatDescr_t, cusparseConstDnMatDescr_t, const void*,
                                                          cusparseSpMatDescr_t, cudaDataType, cusparseSDDMMAlg_t, size_t*);
B200SPMV_EXPORT cusparseStatus_t cusparseSDDMM_preprocess(cusparseHandle_t, cusparseOperation_t, cusparseOperation_t, const void*,
                                                          cusparseConstDnMatDescr_t, cusparseConstDnMatDescr_t, const void*,
                                                          cusparseSpMatDescr_t, cudaDataType, cusparseSDDMMAlg_t, void*);
B200SPMV_EXPORT cusparseStatus_t cusparseSDDMM(cusparseHandle_t, cusparseOperation_t, cusparseOperation_t, const void*,
                                               cusparseConstDnMatDescr_t, cusparseConstDnMatDescr_t, const void*,
                                               cusparseSpMatDescr_t, cudaDataType, cusparseSDDMMAlg_t, void*);
/* cusparse.h:5794-5842 -- spsm_csr_example.c */
B200SPMV_EXPORT cusparseStatus_t cusparseSpSM_createDescr(cusparseSpSMDescr_t*);
B200SPMV_EXPORT cusparseStatus_t cusparseSpSM_destroyDescr(cusparseSpSMDescr_t);
B200SPMV_EXPORT cusparseStatus_t cusparseSpSM_bufferSize(cusparseHandle_t, cusparseOperation_t, cusparseOperation_t, const void*,
                                                         cusparseConstSpMatDescr_t, cusparseConstDnMatDescr_t, cusparseDnMatDescr_t,
                                                         cudaDataType, cusparseSpSMAlg_t, cusparseSpSMDescr_t, size_t*);
B200SPMV_EXPORT cusparseStatus_t cusparseSpSM_analysis(cusparseHandle_t, cusparseOperation_t, cusparseOperation_t, const void*,
                                                       cusparseConstSpMatDescr_t, cusparseConstDnMatDescr_t, cusparseDnMatDescr_t,
                                                       cudaDataType, cusparseSpSMAlg_t, cusparseSpSMDescr_t, void*);
B200SPMV_EXPORT cusparseStatus_t cusparseSpSM_solve(cusparseHandle_t, cusparseOperation_t, cusparseOperation_t, const void*,
                                                    cusparseConstSpMatDescr_t, cusparseConstDnMatDescr_t, cusparseDnMatDescr_t,
                                                    cudaDataType, cusparseSpSMAlg_t, cusparseSpSMDescr_t);
B200SPMV_EXPORT cusparseStatus_t cusparseSpSM_updateMatrix(cusparseHandle_t, cusparseSpSMDescr_t, void*, cusparseSpSMUpdate_t);
/* cusparse.h:3263-3276, 4099-4130, 4951-4982 -- coosort_example.c */
B200SPMV_EXPORT cusparseStatus_t cusparseCsr2cscEx2_bufferSize(cusparseHandle_t, int, int, int, const void*, const int*, const int*, void*,
                                                               int*, int*, cudaDataType, cusparseAction_t, cusparseIndexBase_t,
                                                               cusparseCsr2CscAlg_t, size_t*);
B200SPMV_EXPORT cusparseStatus_t cusparseCsr2cscEx2(cusparseHandle_t, int, int, int, const void*, const int*, const int*, void*, int*, int*,
                                                    cudaDataType, cusparseAction_t, cusparseIndexBase_t, cusparseCsr2CscAlg_t, void*);
B200SPMV_EXPORT cusparseStatus_t cusparseXcoosort_bufferSizeExt(cusparseHandle_t, int, int, int, const int*, const int*, size_t*);
B200SPMV_EXPORT cusparseStatus_t cusparseXcoosortByRow(cusparseHandle_t, int, int, int, int*, int*, int*, void*);
B200SPMV_EXPORT cusparseStatus_t cusparseXcoosortByColumn(cusparseHandle_t, int, int, int, int*, int*, int*, void*);
B200SPMV_EXPORT cusparseStatus_t cusparseXcoo2csr(cusparseHandle_t, const int*, int, int, int*, cusparseIndexBase_t);
B200SPMV_EXPORT cusparseStatus_t cusparseXcsr2coo(cusparseHandle_t, const int*, int, int, int*, cusparseIndexBase_t);
B200SPMV_EXPORT cusparseStatus_t cusparseCreateIdentityPermutation(cusparseHandle_t, int, int*);
/* cusparse.h:5622-5663 -- sparse2dense_csr_example.c, dense2sparse_csr_example.c, dense2sparse_blockedell_example.c.  The
 * bufferSize calls and cusparseDenseToSparse_analysis stay the closed library's. */
B200SPMV_EXPORT cusparseStatus_t cusparseSparseToDense(cusparseHandle_t, cusparseConstSpMatDescr_t, cusparseDnMatDescr_t,
                                                       cusparseSparseToDenseAlg_t, void*);
B200SPMV_EXPORT cusparseStatus_t cusparseDenseToSparse_convert(cusparseHandle_t, cusparseConstDnMatDescr_t, cusparseSpMatDescr_t,
                                                               cusparseDenseToSparseAlg_t, void*);
/* cusparse.h:2650-2840 -- gpsvInterleavedBatch_example.c.  bufferSizeExt returns the larger of the closed library's size and
 * ours, so one buffer serves whichever way the solve is routed. */
B200SPMV_EXPORT cusparseStatus_t cusparseSgtsvInterleavedBatch_bufferSizeExt(cusparseHandle_t, int, int, const float*, const float*,
                                                                             const float*, const float*, int, size_t*);
B200SPMV_EXPORT cusparseStatus_t cusparseSgtsvInterleavedBatch(cusparseHandle_t, int, int, float*, float*, float*, float*, int, void*);
B200SPMV_EXPORT cusparseStatus_t cusparseDgtsvInterleavedBatch_bufferSizeExt(cusparseHandle_t, int, int, const double*, const double*,
                                                                             const double*, const double*, int, size_t*);
B200SPMV_EXPORT cusparseStatus_t cusparseDgtsvInterleavedBatch(cusparseHandle_t, int, int, double*, double*, double*, double*, int, void*);
B200SPMV_EXPORT cusparseStatus_t cusparseCgtsvInterleavedBatch_bufferSizeExt(cusparseHandle_t, int, int, const cuComplex*, const cuComplex*,
                                                                             const cuComplex*, const cuComplex*, int, size_t*);
B200SPMV_EXPORT cusparseStatus_t cusparseCgtsvInterleavedBatch(cusparseHandle_t, int, int, cuComplex*, cuComplex*, cuComplex*, cuComplex*,
                                                               int, void*);
B200SPMV_EXPORT cusparseStatus_t cusparseZgtsvInterleavedBatch_bufferSizeExt(cusparseHandle_t, int, int, const cuDoubleComplex*,
                                                                             const cuDoubleComplex*, const cuDoubleComplex*,
                                                                             const cuDoubleComplex*, int, size_t*);
B200SPMV_EXPORT cusparseStatus_t cusparseZgtsvInterleavedBatch(cusparseHandle_t, int, int, cuDoubleComplex*, cuDoubleComplex*,
                                                               cuDoubleComplex*, cuDoubleComplex*, int, void*);
B200SPMV_EXPORT cusparseStatus_t cusparseSgpsvInterleavedBatch_bufferSizeExt(cusparseHandle_t, int, int, const float*, const float*,
                                                                             const float*, const float*, const float*, const float*, int,
                                                                             size_t*);
B200SPMV_EXPORT cusparseStatus_t cusparseSgpsvInterleavedBatch(cusparseHandle_t, int, int, float*, float*, float*, float*, float*, float*,
                                                               int, void*);
B200SPMV_EXPORT cusparseStatus_t cusparseDgpsvInterleavedBatch_bufferSizeExt(cusparseHandle_t, int, int, const double*, const double*,
                                                                             const double*, const double*, const double*, const double*,
                                                                             int, size_t*);
B200SPMV_EXPORT cusparseStatus_t cusparseDgpsvInterleavedBatch(cusparseHandle_t, int, int, double*, double*, double*, double*, double*,
                                                               double*, int, void*);
B200SPMV_EXPORT cusparseStatus_t cusparseCgpsvInterleavedBatch_bufferSizeExt(cusparseHandle_t, int, int, const cuComplex*, const cuComplex*,
                                                                             const cuComplex*, const cuComplex*, const cuComplex*,
                                                                             const cuComplex*, int, size_t*);
B200SPMV_EXPORT cusparseStatus_t cusparseCgpsvInterleavedBatch(cusparseHandle_t, int, int, cuComplex*, cuComplex*, cuComplex*, cuComplex*,
                                                               cuComplex*, cuComplex*, int, void*);
B200SPMV_EXPORT cusparseStatus_t cusparseZgpsvInterleavedBatch_bufferSizeExt(cusparseHandle_t, int, int, const cuDoubleComplex*,
                                                                             const cuDoubleComplex*, const cuDoubleComplex*,
                                                                             const cuDoubleComplex*, const cuDoubleComplex*,
                                                                             const cuDoubleComplex*, int, size_t*);
B200SPMV_EXPORT cusparseStatus_t cusparseZgpsvInterleavedBatch(cusparseHandle_t, int, int, cuDoubleComplex*, cuDoubleComplex*,
                                                               cuDoubleComplex*, cuDoubleComplex*, cuDoubleComplex*, cuDoubleComplex*, int,
                                                               void*);
/* cusparse.h:434-454, 1434-1666, 1942-2100 -- cg_example.c:423-458, bicgstab_example.c:511-543.  Info objects stay real; the shim
 * keeps a side-table entry per info.  bufferSize returns the larger of the closed library's size and ours; C and Z forward.  The
 * closed library declares the _bufferSizeExt variants but does not export them: the shim's take its _bufferSize and widen it. */
B200SPMV_EXPORT cusparseStatus_t cusparseCreateCsrilu02Info(csrilu02Info_t*);
B200SPMV_EXPORT cusparseStatus_t cusparseDestroyCsrilu02Info(csrilu02Info_t);
B200SPMV_EXPORT cusparseStatus_t cusparseCreateCsric02Info(csric02Info_t*);
B200SPMV_EXPORT cusparseStatus_t cusparseDestroyCsric02Info(csric02Info_t);
B200SPMV_EXPORT cusparseStatus_t cusparseXcsrilu02_zeroPivot(cusparseHandle_t, csrilu02Info_t, int*);
B200SPMV_EXPORT cusparseStatus_t cusparseXcsric02_zeroPivot(cusparseHandle_t, csric02Info_t, int*);
B200SPMV_EXPORT cusparseStatus_t cusparseScsrilu02_numericBoost(cusparseHandle_t, csrilu02Info_t, int, double*, float*);
B200SPMV_EXPORT cusparseStatus_t cusparseDcsrilu02_numericBoost(cusparseHandle_t, csrilu02Info_t, int, double*, double*);
B200SPMV_EXPORT cusparseStatus_t cusparseCcsrilu02_numericBoost(cusparseHandle_t, csrilu02Info_t, int, double*, cuComplex*);
B200SPMV_EXPORT cusparseStatus_t cusparseZcsrilu02_numericBoost(cusparseHandle_t, csrilu02Info_t, int, double*, cuDoubleComplex*);
B200SPMV_EXPORT cusparseStatus_t cusparseScsrilu02_bufferSize(cusparseHandle_t, int, int, const cusparseMatDescr_t, float*, const int*,
                                                              const int*, csrilu02Info_t, int*);
B200SPMV_EXPORT cusparseStatus_t cusparseDcsrilu02_bufferSize(cusparseHandle_t, int, int, const cusparseMatDescr_t, double*, const int*,
                                                              const int*, csrilu02Info_t, int*);
B200SPMV_EXPORT cusparseStatus_t cusparseCcsrilu02_bufferSize(cusparseHandle_t, int, int, const cusparseMatDescr_t, cuComplex*,
                                                              const int*, const int*, csrilu02Info_t, int*);
B200SPMV_EXPORT cusparseStatus_t cusparseZcsrilu02_bufferSize(cusparseHandle_t, int, int, const cusparseMatDescr_t, cuDoubleComplex*,
                                                              const int*, const int*, csrilu02Info_t, int*);
B200SPMV_EXPORT cusparseStatus_t cusparseScsrilu02_bufferSizeExt(cusparseHandle_t, int, int, const cusparseMatDescr_t, float*,
                                                                 const int*, const int*, csrilu02Info_t, size_t*);
B200SPMV_EXPORT cusparseStatus_t cusparseDcsrilu02_bufferSizeExt(cusparseHandle_t, int, int, const cusparseMatDescr_t, double*,
                                                                 const int*, const int*, csrilu02Info_t, size_t*);
B200SPMV_EXPORT cusparseStatus_t cusparseCcsrilu02_bufferSizeExt(cusparseHandle_t, int, int, const cusparseMatDescr_t, cuComplex*,
                                                                 const int*, const int*, csrilu02Info_t, size_t*);
B200SPMV_EXPORT cusparseStatus_t cusparseZcsrilu02_bufferSizeExt(cusparseHandle_t, int, int, const cusparseMatDescr_t, cuDoubleComplex*,
                                                                 const int*, const int*, csrilu02Info_t, size_t*);
B200SPMV_EXPORT cusparseStatus_t cusparseScsrilu02_analysis(cusparseHandle_t, int, int, const cusparseMatDescr_t, const float*,
                                                            const int*, const int*, csrilu02Info_t, cusparseSolvePolicy_t, void*);
B200SPMV_EXPORT cusparseStatus_t cusparseDcsrilu02_analysis(cusparseHandle_t, int, int, const cusparseMatDescr_t, const double*,
                                                            const int*, const int*, csrilu02Info_t, cusparseSolvePolicy_t, void*);
B200SPMV_EXPORT cusparseStatus_t cusparseCcsrilu02_analysis(cusparseHandle_t, int, int, const cusparseMatDescr_t, const cuComplex*,
                                                            const int*, const int*, csrilu02Info_t, cusparseSolvePolicy_t, void*);
B200SPMV_EXPORT cusparseStatus_t cusparseZcsrilu02_analysis(cusparseHandle_t, int, int, const cusparseMatDescr_t, const cuDoubleComplex*,
                                                            const int*, const int*, csrilu02Info_t, cusparseSolvePolicy_t, void*);
B200SPMV_EXPORT cusparseStatus_t cusparseScsrilu02(cusparseHandle_t, int, int, const cusparseMatDescr_t, float*, const int*, const int*,
                                                   csrilu02Info_t, cusparseSolvePolicy_t, void*);
B200SPMV_EXPORT cusparseStatus_t cusparseDcsrilu02(cusparseHandle_t, int, int, const cusparseMatDescr_t, double*, const int*, const int*,
                                                   csrilu02Info_t, cusparseSolvePolicy_t, void*);
B200SPMV_EXPORT cusparseStatus_t cusparseCcsrilu02(cusparseHandle_t, int, int, const cusparseMatDescr_t, cuComplex*, const int*,
                                                   const int*, csrilu02Info_t, cusparseSolvePolicy_t, void*);
B200SPMV_EXPORT cusparseStatus_t cusparseZcsrilu02(cusparseHandle_t, int, int, const cusparseMatDescr_t, cuDoubleComplex*, const int*,
                                                   const int*, csrilu02Info_t, cusparseSolvePolicy_t, void*);
B200SPMV_EXPORT cusparseStatus_t cusparseScsric02_bufferSize(cusparseHandle_t, int, int, const cusparseMatDescr_t, float*, const int*,
                                                             const int*, csric02Info_t, int*);
B200SPMV_EXPORT cusparseStatus_t cusparseDcsric02_bufferSize(cusparseHandle_t, int, int, const cusparseMatDescr_t, double*, const int*,
                                                             const int*, csric02Info_t, int*);
B200SPMV_EXPORT cusparseStatus_t cusparseCcsric02_bufferSize(cusparseHandle_t, int, int, const cusparseMatDescr_t, cuComplex*,
                                                             const int*, const int*, csric02Info_t, int*);
B200SPMV_EXPORT cusparseStatus_t cusparseZcsric02_bufferSize(cusparseHandle_t, int, int, const cusparseMatDescr_t, cuDoubleComplex*,
                                                             const int*, const int*, csric02Info_t, int*);
B200SPMV_EXPORT cusparseStatus_t cusparseScsric02_bufferSizeExt(cusparseHandle_t, int, int, const cusparseMatDescr_t, float*,
                                                                const int*, const int*, csric02Info_t, size_t*);
B200SPMV_EXPORT cusparseStatus_t cusparseDcsric02_bufferSizeExt(cusparseHandle_t, int, int, const cusparseMatDescr_t, double*,
                                                                const int*, const int*, csric02Info_t, size_t*);
B200SPMV_EXPORT cusparseStatus_t cusparseCcsric02_bufferSizeExt(cusparseHandle_t, int, int, const cusparseMatDescr_t, cuComplex*,
                                                                const int*, const int*, csric02Info_t, size_t*);
B200SPMV_EXPORT cusparseStatus_t cusparseZcsric02_bufferSizeExt(cusparseHandle_t, int, int, const cusparseMatDescr_t, cuDoubleComplex*,
                                                                const int*, const int*, csric02Info_t, size_t*);
B200SPMV_EXPORT cusparseStatus_t cusparseScsric02_analysis(cusparseHandle_t, int, int, const cusparseMatDescr_t, const float*,
                                                           const int*, const int*, csric02Info_t, cusparseSolvePolicy_t, void*);
B200SPMV_EXPORT cusparseStatus_t cusparseDcsric02_analysis(cusparseHandle_t, int, int, const cusparseMatDescr_t, const double*,
                                                           const int*, const int*, csric02Info_t, cusparseSolvePolicy_t, void*);
B200SPMV_EXPORT cusparseStatus_t cusparseCcsric02_analysis(cusparseHandle_t, int, int, const cusparseMatDescr_t, const cuComplex*,
                                                           const int*, const int*, csric02Info_t, cusparseSolvePolicy_t, void*);
B200SPMV_EXPORT cusparseStatus_t cusparseZcsric02_analysis(cusparseHandle_t, int, int, const cusparseMatDescr_t, const cuDoubleComplex*,
                                                           const int*, const int*, csric02Info_t, cusparseSolvePolicy_t, void*);
B200SPMV_EXPORT cusparseStatus_t cusparseScsric02(cusparseHandle_t, int, int, const cusparseMatDescr_t, float*, const int*, const int*,
                                                  csric02Info_t, cusparseSolvePolicy_t, void*);
B200SPMV_EXPORT cusparseStatus_t cusparseDcsric02(cusparseHandle_t, int, int, const cusparseMatDescr_t, double*, const int*, const int*,
                                                  csric02Info_t, cusparseSolvePolicy_t, void*);
B200SPMV_EXPORT cusparseStatus_t cusparseCcsric02(cusparseHandle_t, int, int, const cusparseMatDescr_t, cuComplex*, const int*,
                                                  const int*, csric02Info_t, cusparseSolvePolicy_t, void*);
B200SPMV_EXPORT cusparseStatus_t cusparseZcsric02(cusparseHandle_t, int, int, const cusparseMatDescr_t, cuDoubleComplex*, const int*,
                                                  const int*, csric02Info_t, cusparseSolvePolicy_t, void*);
/* cusparse.h:5917-5920, 6019-6041 -- spgemm_reuse_example.c.  The descriptor stays the closed library's; the shim keeps a side-table
 * entry per descriptor.  cusparseSpGEMMreuse_workEstimation / _nnz and the whole non-reuse SpGEMM API are not exported: they bind
 * to the closed library. */
B200SPMV_EXPORT cusparseStatus_t cusparseSpGEMM_createDescr(cusparseSpGEMMDescr_t*);
B200SPMV_EXPORT cusparseStatus_t cusparseSpGEMM_destroyDescr(cusparseSpGEMMDescr_t);
B200SPMV_EXPORT cusparseStatus_t cusparseSpGEMMreuse_copy(cusparseHandle_t, cusparseOperation_t, cusparseOperation_t, cusparseConstSpMatDescr_t,
                                                          cusparseConstSpMatDescr_t, cusparseSpMatDescr_t, cusparseSpGEMMAlg_t,
                                                          cusparseSpGEMMDescr_t, size_t*, void*);
B200SPMV_EXPORT cusparseStatus_t cusparseSpGEMMreuse_compute(cusparseHandle_t, cusparseOperation_t, cusparseOperation_t, const void*,
                                                             cusparseConstSpMatDescr_t, cusparseConstSpMatDescr_t, const void*,
                                                             cusparseSpMatDescr_t, cudaDataType, cusparseSpGEMMAlg_t, cusparseSpGEMMDescr_t);
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
