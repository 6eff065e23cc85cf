/*
 * b200spsv.h -- C ABI of libb200spsv.so, the H100-native (sm_90a) CSR triangular solve behind cusparseSpSV_*
 * (NVIDIA/CUDALibrarySamples cuSPARSE/spsv_csr, and the preconditioner solves of cuSPARSE/cg and cuSPARSE/bicgstab).
 *
 * A library of its own, next to libb200spmv.so, so that opting in is a link-order decision:
 *
 *     -lb200spsv -lb200spmv -lcusparse      SpSV and SpMV native, everything else closed
 *     -lb200spmv -lcusparse                 SpMV native, SpSV closed (libb200spmv.so exports no cusparseSpSV_*)
 *     LD_PRELOAD=libb200spsv.so ./stock     SpSV native in a binary linked against libcusparse only
 *
 * It does not depend on libb200spmv.so: it reaches the real libcusparse.so.12 through dlopen (B200SPMV_CUSPARSE, then the
 * usual sonames) and reads matrix descriptors through the real getters, whoever created them.
 *
 * Two layers, both `extern "C"`:
 *   1. cusparseSpSV_createDescr / _destroyDescr / _bufferSize / _analysis / _solve / _updateMatrix with the exact
 *      prototypes of cusparse.h (CUDA 12.9, cusparse.h:5729-5774); compile with -DB200SPSV_DECLARE_CUSPARSE to see them.
 *   2. The native entry points underneath (b200spsv_*): descriptor-free, usable without libcusparse.
 *
 * Every exported function is tagged B200SPSV_EXPORT.
 */
#ifndef B200SPSV_H_
#define B200SPSV_H_

#include <stddef.h>
#include <stdint.h>

#define B200SPSV_EXPORT /* exported from libb200spsv.so */

#ifdef __cplusplus
extern "C" {
#endif

/* ============================================================================================== *
 * Layer 2: native entry points.                                                                   *
 *   Solves op(T) y = alpha x, T the selected triangle of the rows x rows CSR matrix A (int32      *
 *   offsets and columns, index base 0 or 1).  A may store both triangles: entries outside the      *
 *   selected one are ignored, and with unit = 1 so is the stored diagonal.                        *
 *   lower     : 1 = T is the lower triangle of A (CUSPARSE_FILL_MODE_LOWER), 0 = the upper one     *
 *   unit      : 1 = unit diagonal (CUSPARSE_DIAG_TYPE_UNIT), 0 = divide by the stored diagonal     *
 *   transpose : 0 = solve with T, 1 = with T^T                                                    *
 *   dtype     : 0 = fp32, 1 = fp64 (values, x, y, alpha and the arithmetic)                       *
 *   return    : 0 on success, -1 on invalid arguments (checked before any CUDA call), otherwise   *
 *               the cudaError_t of the failing CUDA call.                                         *
 * ============================================================================================== */

/* Bytes of the workspace _analysis builds the solve plan in.  The same workspace must be passed to every
 * _solve of that plan; it also holds the solve-state words, so two solves of one plan must not overlap. */
B200SPSV_EXPORT size_t b200spsv_csr_workspace_bytes(int64_t rows, int64_t nnz, int transpose);

/* Byte offsets of the plan's arrays inside the workspace (each 256-byte aligned), for tests and tools:
 *   offsets[B200SPSV_STATE]  uint32 state words: [0] epoch of the last solve, [1] rows claimed by it,
 *                            [2] error word (0 = no wait ran out of budget), [3] rows without a stored diagonal
 *                            (counted for unit = 0 only)
 *   offsets[B200SPSV_FLAGS]  uint32[rows]: row i is solved when flags[i] == epoch
 *   offsets[B200SPSV_T_OFF]  int32[rows + 1]: row offsets of op(T) without its diagonal
 *   offsets[B200SPSV_DIAG]   int32[rows]: index into values of the diagonal of row i, -1 for unit = 1 or none stored
 *   offsets[B200SPSV_T_COL]  int32[t_off[rows]]: the row of y each entry depends on
 *   offsets[B200SPSV_T_VIDX] int32[t_off[rows]]: index of the entry in the caller's values (0-based)
 *   offsets[B200SPSV_SCRATCH] analysis scratch;  offsets[B200SPSV_TOTAL] == b200spsv_csr_workspace_bytes(...)
 * Entries of a plan row are in stored order (transpose = 0) or ascending row of A (transpose = 1).
 * Returns -1 for negative sizes. */
enum { B200SPSV_STATE = 0, B200SPSV_FLAGS, B200SPSV_T_OFF, B200SPSV_DIAG, B200SPSV_T_COL, B200SPSV_T_VIDX, B200SPSV_SCRATCH,
       B200SPSV_TOTAL, B200SPSV_LAYOUT_N };
B200SPSV_EXPORT int b200spsv_csr_layout(int64_t rows, int64_t nnz, int transpose, size_t* offsets /* [B200SPSV_LAYOUT_N] */);

/* Builds the plan (integer work only; values are not read) and clears the state words.  When missing_diag is not NULL,
 * the number of rows without a stored diagonal (unit = 0) is copied into it, which synchronises the stream once;
 * with NULL the call is asynchronous. */
B200SPSV_EXPORT int b200spsv_csr_analysis(void* stream, int64_t rows, int64_t nnz, const void* row_offsets, const void* col_ind,
                                          int32_t base, int lower, int unit, int transpose, void* workspace,
                                          int64_t* missing_diag);

/* op(T) y = alpha x with the plan in workspace (built by _analysis with the same rows, nnz, lower, unit, transpose).
 * values are read now; diag (rows values of dtype, or NULL) replaces the stored diagonal.  alpha is a host pointer
 * (alpha_on_device = 0) or a device pointer read inside the kernel.  x may equal y.  Two launches on stream, no
 * allocation, no host synchronisation: CUDA-graph capturable. */
B200SPSV_EXPORT int b200spsv_csr_solve(void* stream, int dtype, int64_t rows, int64_t nnz, int lower, int unit, int transpose,
                                       const void* values, const void* diag, const void* alpha, int alpha_on_device,
                                       const void* x, void* y, void* workspace);

/* Threads per CTA of the solve kernel, and the budget in nanoseconds (%globaltimer) of any one wait for a dependency:
 * a wait that runs out sets the error word, the row is written as NaN and the solve runs to its end. */
B200SPSV_EXPORT void b200spsv_csr_params(int32_t* threads_per_cta, uint64_t* spin_budget_ns);

/* Would cusparseSpSV_analysis serve a call of this shape natively?  1: yes (the analysis may still forward a NON_UNIT
 * matrix with a row that stores no diagonal), 0: handed to the closed library.  Pure host logic. */
B200SPSV_EXPORT int b200spsv_route(int format, int op, int alg, int off_type, int col_type, int a_vtype, int x_vtype, int y_vtype,
                                   int compute_type, int fill, int diag, int64_t rows, int64_t cols, int64_t nnz);

/* Since the last reset: solves run natively / SpSV calls handed to the closed library / native analyses. */
B200SPSV_EXPORT void b200spsv_get_stats(uint64_t* native_calls, uint64_t* forwarded_calls, uint64_t* analysis_calls);
B200SPSV_EXPORT void b200spsv_reset_stats(void);
B200SPSV_EXPORT const char* b200spsv_version(void);

#ifdef __cplusplus
}
#endif

/* ============================================================================================== *
 * Layer 1: the cuSPARSE symbols (prototypes == cusparse.h of CUDA 12.9).                          *
 * ============================================================================================== */
#ifdef B200SPSV_DECLARE_CUSPARSE
#include <cusparse.h>
#ifdef __cplusplus
extern "C" {
#endif
/* cusparse.h:5730 / 5733 -- spsv_csr_example.c:97,126, cg_example.c:167,184,302-303 */
B200SPSV_EXPORT cusparseStatus_t cusparseSpSV_createDescr(cusparseSpSVDescr_t*);
B200SPSV_EXPORT cusparseStatus_t cusparseSpSV_destroyDescr(cusparseSpSVDescr_t);
/* cusparse.h:5736 -- spsv_csr_example.c:107-111 */
B200SPSV_EXPORT cusparseStatus_t cusparseSpSV_bufferSize(cusparseHandle_t, cusparseOperation_t, const void*, cusparseConstSpMatDescr_t,
                                                         cusparseConstDnVecDescr_t, cusparseDnVecDescr_t, cudaDataType,
                                                         cusparseSpSVAlg_t, cusparseSpSVDescr_t, size_t*);
/* cusparse.h:5748 -- spsv_csr_example.c:113-116 */
B200SPSV_EXPORT cusparseStatus_t cusparseSpSV_analysis(cusparseHandle_t, cusparseOperation_t, const void*, cusparseConstSpMatDescr_t,
                                                       cusparseConstDnVecDescr_t, cusparseDnVecDescr_t, cudaDataType,
                                                       cusparseSpSVAlg_t, cusparseSpSVDescr_t, void*);
/* cusparse.h:5760 -- spsv_csr_example.c:118-120, cg_example.c:256,263, bicgstab_example.c:246-306 */
B200SPSV_EXPORT cusparseStatus_t cusparseSpSV_solve(cusparseHandle_t, cusparseOperation_t, const void*, cusparseConstSpMatDescr_t,
                                                    cusparseConstDnVecDescr_t, cusparseDnVecDescr_t, cudaDataType,
                                                    cusparseSpSVAlg_t, cusparseSpSVDescr_t);
/* cusparse.h:5771 */
B200SPSV_EXPORT cusparseStatus_t cusparseSpSV_updateMatrix(cusparseHandle_t, cusparseSpSVDescr_t, void*, cusparseSpSVUpdate_t);
#ifdef __cplusplus
}
#endif
#endif /* B200SPSV_DECLARE_CUSPARSE */

#endif /* B200SPSV_H_ */
