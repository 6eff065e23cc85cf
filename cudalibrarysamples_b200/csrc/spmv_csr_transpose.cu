// spmv_csr_transpose.cu -- CSR  y = alpha*A^T*x + beta*y  on H100 (sm_90a): opA = CUSPARSE_OPERATION_TRANSPOSE (and
// CONJUGATE_TRANSPOSE, the same thing for real types) of cusparseSpMV on CSR descriptors (SURVEY.md 8(f)-3; formerly
// forwarded to the closed library).  A is rows x cols, x has `rows` entries, y has `cols` entries.
//
// A^T in CSR storage is a scatter: non-zero (r, c, v) adds alpha*v*x[r] to y[c].  Two launches:
//   1. y = beta*y (beta == 0: plain zero fill, y is never read; beta == 1: skipped when beta is known on the host);
//   2. csr_transpose_kernel: every warp owns 256 consecutive non-zeros -- coalesced loads of col_ind / val as in the other
//      CSR kernels; the row of the warp's first non-zero comes from one binary search over row_offsets, after that every
//      lane walks forward through the (L1-resident) offsets as its element index grows; x[r] is a broadcast-like load
//      (neighbouring lanes share rows), the result goes out as one RED.ADD per non-zero (fp atomics at L2).
// The summation order of a column is not fixed -> results agree with the oracle to tolerance, not bit for bit; the closed
// library makes no reproducibility promise for opA != NON_TRANSPOSE either (cusparse.h, cusparseSpMVAlg_t notes).
// Bytes: nnz*(val+4) + (rows+1)*4 + rows*val (x) + 2*cols*val (y read-modify-write by the atomics).
#include "spmv_common.cuh"
#include "config.h"
#include "../../include/b200spmv.h"

namespace b200 {

constexpr int TR_BLOCK = 256;
constexpr int TR_STEPS = 8;                      // 32-element steps per warp chunk
constexpr int TR_CHUNK = 32 * TR_STEPS;

template <typename T>
struct TrArgs {
    const int* off;
    const int* col;
    const T*   val;
    const T*   x;
    T*         y;
    int        base, rows, cols, nnz;
    Scalars<T> s;
};

template <typename T>
__global__ void tr_scale_y_kernel(T* __restrict__ y, int64_t n, Scalars<T> s) {
    const T beta = s.b();
    if (beta == T(1)) return;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
        y[i] = beta == T(0) ? T(0) : beta * y[i];
}

template <typename T>
__global__ void __launch_bounds__(TR_BLOCK) csr_transpose_kernel(const TrArgs<T> a) {
    const int lane = (int)threadIdx.x & 31;
    const long long wid = (long long)blockIdx.x * (TR_BLOCK / 32) + ((int)threadIdx.x >> 5);
    const long long c0 = wid * TR_CHUNK;
    if (c0 >= a.nnz) return;                                       // warp-uniform
    const int n0 = (int)c0, n1 = min(n0 + TR_CHUNK, a.nnz);
    const T alpha = a.s.a();
    int r = csr_row_of(a.off, a.rows, a.base, n0);
    int rend = __ldg(a.off + r + 1) - a.base;                      // first non-zero behind my current row
    int cc[TR_STEPS];
    T   vv[TR_STEPS];
#pragma unroll
    for (int k = 0; k < TR_STEPS; k++) {
        const int i = n0 + k * 32 + lane;
        const bool live = i < n1;
        cc[k] = live ? ldg_stream(a.col + i) : a.base;
        vv[k] = live ? ldg_stream(a.val + i) : T(0);
    }
#pragma unroll
    for (int k = 0; k < TR_STEPS; k++) {
        const int i = n0 + k * 32 + lane;
        if (i < n1) {
            while (rend <= i) { r++; rend = __ldg(a.off + r + 1) - a.base; }     // i < nnz = off[rows] - base: stops at r < rows
            atomicAdd(a.y + (cc[k] - a.base), alpha * vv[k] * __ldg(a.x + r));
        }
    }
}

template <typename T>
static int launch_transpose(cudaStream_t stream, int64_t rows, int64_t cols, int64_t nnz, const void* off, const void* col,
                            const void* val, int base, const void* alpha, const void* beta, int on_device, const void* x, void* y) {
    TrArgs<T> a;
    a.off = (const int*)off; a.col = (const int*)col; a.val = (const T*)val; a.x = (const T*)x; a.y = (T*)y;
    a.base = base; a.rows = (int)rows; a.cols = (int)cols; a.nnz = (int)nnz;
    set_scalars(a.s, alpha, beta, on_device);
    stats().last_csr_kernel = sizeof(T) == 8 ? "b200::csr_transpose_kernel<double>" : "b200::csr_transpose_kernel<float>";
    if (cols > 0 && (on_device || *(const T*)beta != T(1))) {
        int64_t blocks = (cols + 255) / 256;
        if (blocks > 132 * 16) blocks = 132 * 16;
        tr_scale_y_kernel<T><<<(unsigned)blocks, 256, 0, stream>>>((T*)y, cols, a.s);
        cudaError_t e = cudaGetLastError();
        if (e != cudaSuccess) return (int)e;
    }
    if (nnz == 0 || rows == 0) return 0;
    const int64_t warps = (nnz + TR_CHUNK - 1) / TR_CHUNK;
    const int64_t ctas = (warps + TR_BLOCK / 32 - 1) / (TR_BLOCK / 32);
    csr_transpose_kernel<T><<<(unsigned)ctas, TR_BLOCK, 0, stream>>>(a);
    return (int)cudaGetLastError();
}

}  // namespace b200

using namespace b200;

extern "C" int b200spmv_csr_transpose_mv(void* stream, int dtype, int64_t rows, int64_t cols, int64_t nnz, const void* row_offsets,
                                         const void* col_ind, const void* values, int32_t base, const void* alpha, const void* beta,
                                         int scalars_on_device, const void* x, void* y) {
    if (rows < 0 || cols < 0 || nnz < 0 || !alpha || !beta) return -1;
    if (cols == 0) return 0;
    if (rows > INT32_MAX - 64 || cols > INT32_MAX - 64 || nnz > INT32_MAX - 65536) return -1;
    if (!y || (rows > 0 && !row_offsets) || (nnz > 0 && (!col_ind || !values || !x))) return -1;
    if (dtype == 0)
        return launch_transpose<float>((cudaStream_t)stream, rows, cols, nnz, row_offsets, col_ind, values, base, alpha, beta, scalars_on_device, x, y);
    if (dtype == 1)
        return launch_transpose<double>((cudaStream_t)stream, rows, cols, nnz, row_offsets, col_ind, values, base, alpha, beta, scalars_on_device, x, y);
    return -1;
}
