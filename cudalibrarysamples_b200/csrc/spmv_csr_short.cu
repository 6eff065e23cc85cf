// spmv_csr_short.cu -- CSR  y = alpha*A*x + beta*y  on H100 (sm_90a) for matrices whose rows are ALL short (stencils,
// meshes: 5-pt Poisson of cuSPARSE/cg/cg_example.c:71-128, 7-pt Laplacian of cuDSS/simple_residual/laplace_generator.hxx).
//
// Why a third CSR path: on the 5-pt / 7-pt operators the tile / pipe kernels stay well below the HBM roofline while the
// Sliced-ELL kernel runs the SAME operator close to it -- the difference is the row bookkeeping: merge-path tiles, a CTA-wide barrier between the load and
// the reduce phase, lane groups + shuffle trees for rows of 5-7 elements.  With short rows none of that is needed:
//
//   a warp owns 32 consecutive rows = one contiguous range [b, e) of non-zeros (about 160-220 for the stencils);
//   it streams col_ind / val over that range with coalesced 128 B / 256 B loads (the range start is rounded down to a
//   multiple of 32 elements so every warp-level load is line-aligned), gathers x, parks the products in its own slice of
//   shared memory (skewed by one slot per 32: the row-strided reads below are bank-conflict free for every row length),
//   __syncwarp, and then lane l adds up row l's products serially -- a fixed, sequential order per row: bit-reproducible.
//   No CTA barrier, no shuffles, no plan: the kernel reads the caller's
//   row offsets directly.  Ranges longer than the per-warp buffer are walked in passes (correct for any row length);
//   cusparseSpMV_preprocess selects this kernel only when the longest row has at most SHORT_MAX_ROW non-zeros.
//
// Bytes per launch = the CSR algorithmic bytes (SURVEY.md 8d); bound: HBM.
// Replaces cusparse::csrmv_v3_kernel behind cusparseSpMV for preprocessed CSR descriptors with short rows
// (call sites: cuSPARSE/cg/cg_example.c:156-160,220-224; cuSPARSE/bicgstab/bicgstab_example.c:175-180).
#include "spmv_common.cuh"
#include "config.h"
#include "../../include/b200spmv.h"

namespace b200 {

#ifndef B200_SHORT_WARPS
#define B200_SHORT_WARPS 8          // warps (= 32-row blocks) per CTA
#endif
#ifndef B200_SHORT_STEPS
#define B200_SHORT_STEPS 8          // 32-element load steps per pass: the per-warp buffer holds 32 * STEPS products
#endif
#ifndef B200_SHORT_MIN_CTAS
#define B200_SHORT_MIN_CTAS 5       // fp64 (48 registers); fp32 runs one more CTA per SM (40 registers) -- swept on an earlier GPU, not re-swept on the H100 (scripts/sweep.py SHORT)
#endif
constexpr int SHORT_WARPS = B200_SHORT_WARPS;
constexpr int SHORT_STEPS = B200_SHORT_STEPS;
constexpr int SHORT_CAP = 32 * SHORT_STEPS;             // products per pass
constexpr int SHORT_SLOTS = SHORT_CAP + SHORT_STEPS;    // + one skew slot per 32
constexpr int SHORT_MAX_ROW = 32;                       // preprocess picks this kernel up to this row length

template <typename T>
struct ShortArgs {
    const int* off;
    const int* col;
    const T*   val;
    const T*   x;
    T*         y;
    int        base, rows;
    Scalars<T> s;
    // DOT variant (SURVEY.md 8(f)-2, "fuse dot(T, P) into the SpMV epilogue", cg_example.c:220-227): *dot_out = sum_i y[i] * w[i]
    const T*   w;
    double*    dot_ws;     // one partial per CTA, then the arrival counter
    double*    dot_out;
};

__device__ __forceinline__ int short_slot(int i) { return i + (i >> 5); }

constexpr int SHORT_MAX_GRID = 132 * (B200_SHORT_MIN_CTAS + 1) * 8;     // launch_short never starts more CTAs than this

template <typename T, bool DOT>
__global__ void __launch_bounds__(32 * SHORT_WARPS, (sizeof(T) == 8 ? B200_SHORT_MIN_CTAS : B200_SHORT_MIN_CTAS + 1))
csr_short_kernel(const ShortArgs<T> a) {
    __shared__ T sprod[SHORT_WARPS][SHORT_SLOTS];
    double dsum = 0.0;                                        // DOT: this lane's share of y . w
    const int lane = (int)threadIdx.x & 31, warp = (int)threadIdx.x >> 5;
    T* sp = sprod[warp];
    const T alpha = a.s.a(), beta = a.s.b();
    const int nblocks = (int)(((long long)a.rows + 31) >> 5);                    // no int overflow for rows near INT32_MAX
    for (int blk = blockIdx.x * SHORT_WARPS + warp; blk < nblocks; blk += gridDim.x * SHORT_WARPS) {   // warp-uniform
        const int row = (blk << 5) + lane;
        const bool live = row < a.rows;
        const int rb = __ldg(a.off + min(row, a.rows)) - a.base;                  // (rows past the end: empty, at nnz)
        const int re = live ? __ldg(a.off + row + 1) - a.base : rb;
        const int b = __shfl_sync(0xffffffffu, rb, 0);
        const int e = __shfl_sync(0xffffffffu, re, 31);                           // lanes past the last row carry its end
        T sum = T(0);
        // passes over [b, e), starting at a multiple of 32 elements (line-aligned warp loads; the elements in front of b
        // belong to earlier rows: loaded, multiplied, never read back)
        for (int p0 = b & ~31; p0 < e; p0 += SHORT_CAP) {
            int cc[SHORT_STEPS];
            T   vv[SHORT_STEPS];
#pragma unroll
            for (int k = 0; k < SHORT_STEPS; k++) {
                const int i = p0 + k * 32 + lane;
                const bool in = i < e;
                cc[k] = in ? ldg_stream(a.col + i) : a.base;
                vv[k] = in ? ldg_stream(a.val + i) : T(0);
            }
            const T* xp = a.x - a.base;
#pragma unroll
            for (int k = 0; k < SHORT_STEPS; k++) {
                if (p0 + k * 32 < e)                                              // warp-uniform
                    sp[short_slot(k * 32 + lane)] = vv[k] * __ldg(xp + cc[k]);
            }
            __syncwarp();
            const int lo = max(rb, p0) - p0, hi = min(re, p0 + SHORT_CAP) - p0;   // my row's part of this pass
            for (int i = lo; i < hi; i++) sum += sp[short_slot(i)];
            __syncwarp();
        }
        if (live) {
            const T yv = axpby(alpha, sum, beta, a.y + row);
            a.y[row] = yv;
            if (DOT) dsum += (double)yv * (double)__ldg(a.w + row);
        }
    }
    if (DOT) {
        // deterministic three-level sum: lanes (butterfly), warps of the CTA (in warp order), CTAs (in CTA order, by the CTA
        // that arrives last) -- same scheme as csrc/cg_fused.cu
        __shared__ double swarp[SHORT_WARPS];
        dsum = warp_allsum(dsum);
        if (lane == 0) swarp[warp] = dsum;
        __syncthreads();
        if (threadIdx.x == 0) {
            double part = 0.0;
#pragma unroll
            for (int w = 0; w < SHORT_WARPS; w++) part += swarp[w];
            unsigned* counter = (unsigned*)(a.dot_ws + SHORT_MAX_GRID);
            a.dot_ws[blockIdx.x] = part;
            __threadfence();
            if (atomicAdd(counter, 1u) == gridDim.x - 1) {
                __threadfence();
                double t = 0.0;
                for (unsigned b = 0; b < gridDim.x; b++) t += __ldcg(a.dot_ws + b);
                *a.dot_out = t;
                *counter = 0u;
            }
        }
    }
}

// longest row of the matrix (structure-only statistic read back once by cusparseSpMV_preprocess)
__global__ void csr_max_row_kernel(const int* __restrict__ off, int64_t rows, int* __restrict__ out) {
    int m = 0;
    for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < rows; r += (int64_t)gridDim.x * blockDim.x)
        m = max(m, off[r + 1] - off[r]);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) m = max(m, __shfl_xor_sync(0xffffffffu, m, o));
    if ((threadIdx.x & 31) == 0 && m > 0) atomicMax(out, m);
}

template <typename T>
static int launch_short(cudaStream_t stream, int64_t rows, const void* off, const void* col, const void* val, int base,
                        const void* alpha, const void* beta, int on_device, const void* x, void* y,
                        const void* w = nullptr, double* dot_out = nullptr, void* dot_ws = nullptr) {
    ShortArgs<T> a;
    a.w = (const T*)w; a.dot_out = dot_out; a.dot_ws = (double*)dot_ws;
    a.off = (const int*)off; a.col = (const int*)col; a.val = (const T*)val; a.x = (const T*)x; a.y = (T*)y;
    a.base = base; a.rows = (int)rows;
    set_scalars(a.s, alpha, beta, on_device);
    stats().last_csr_kernel = sizeof(T) == 8 ? "b200::csr_short_kernel<double>" : "b200::csr_short_kernel<float>";
    const int64_t nblocks = (rows + 31) / 32;
    int64_t ctas = (nblocks + SHORT_WARPS - 1) / SHORT_WARPS;
    const int64_t cap = 132LL * (B200_SHORT_MIN_CTAS + (sizeof(T) == 8 ? 0 : 1)) * 8;      // a few waves; beyond that the warps loop
    if (ctas > cap) ctas = cap;
    if (dot_out) csr_short_kernel<T, true><<<(unsigned)ctas, 32 * SHORT_WARPS, 0, stream>>>(a);
    else         csr_short_kernel<T, false><<<(unsigned)ctas, 32 * SHORT_WARPS, 0, stream>>>(a);
    return (int)cudaGetLastError();
}

}  // namespace b200

using namespace b200;

extern "C" {

int b200spmv_csr_short_max_row(void) { return SHORT_MAX_ROW; }

void b200spmv_csr_short_params(int32_t* pass_cap, int32_t* rows_per_warp) {
    if (pass_cap) *pass_cap = SHORT_CAP;
    if (rows_per_warp) *rows_per_warp = 32;
}

int b200spmv_csr_max_row_length(void* stream, int64_t rows, const void* row_offsets, int32_t* out_device) {
    if (rows < 0 || !out_device || (rows > 0 && !row_offsets)) return -1;
    cudaStream_t st = (cudaStream_t)stream;
    cudaError_t e = cudaMemsetAsync(out_device, 0, sizeof(int32_t), st);
    if (e != cudaSuccess) return (int)e;
    if (rows == 0) return 0;
    int64_t blocks = (rows + 255) / 256;
    if (blocks > 132 * 16) blocks = 132 * 16;
    csr_max_row_kernel<<<(unsigned)blocks, 256, 0, st>>>((const int*)row_offsets, rows, out_device);
    return (int)cudaGetLastError();
}

// y = alpha*A*x + beta*y and, in the same pass, *dot_out = y . w (device memory, fp64 accumulation): the T = A*P product of a
// CG iteration together with its T . P (cg_example.c:220-227).  workspace: b200spmv_csr_short_dot_workspace_bytes(),
// zeroed once before first use; every call leaves the arrival counter at zero.
size_t b200spmv_csr_short_dot_workspace_bytes(void) { return (size_t)(SHORT_MAX_GRID + 2) * sizeof(double); }

int b200spmv_csr_short_mv_dot(void* stream, int dtype, int64_t rows, int64_t cols, int64_t nnz, const void* row_offsets,
                              const void* col_ind, const void* values, int32_t base, const void* alpha, const void* beta,
                              int scalars_on_device, const void* x, void* y, const void* w, double* dot_out, void* workspace) {
    if (rows < 0 || cols < 0 || nnz < 0 || !alpha || !beta || !dot_out || !workspace) return -1;
    if (rows > INT32_MAX - 64 || nnz > INT32_MAX - 65536) return -1;
    if (rows > 0 && (!y || !w || !row_offsets || (nnz > 0 && (!col_ind || !values || !x)))) return -1;
    if (rows == 0) return (int)cudaMemsetAsync(dot_out, 0, sizeof(double), (cudaStream_t)stream);
    if (dtype == 0)
        return launch_short<float>((cudaStream_t)stream, rows, row_offsets, col_ind, values, base, alpha, beta, scalars_on_device, x, y, w, dot_out, workspace);
    if (dtype == 1)
        return launch_short<double>((cudaStream_t)stream, rows, row_offsets, col_ind, values, base, alpha, beta, scalars_on_device, x, y, w, dot_out, workspace);
    return -1;
}

int b200spmv_csr_short_mv(void* stream, int dtype, int64_t rows, int64_t cols, int64_t nnz, const void* row_offsets,
                          const void* col_ind, const void* values, int32_t base, const void* alpha, const void* beta,
                          int scalars_on_device, const void* x, void* y) {
    if (rows < 0 || cols < 0 || nnz < 0 || !alpha || !beta) return -1;
    if (rows == 0) return 0;
    if (rows > INT32_MAX - 64 || nnz > INT32_MAX - 65536) return -1;
    if (!y || !row_offsets || (nnz > 0 && (!col_ind || !values || !x))) return -1;
    if (dtype == 0)
        return launch_short<float>((cudaStream_t)stream, rows, row_offsets, col_ind, values, base, alpha, beta, scalars_on_device, x, y);
    if (dtype == 1)
        return launch_short<double>((cudaStream_t)stream, rows, row_offsets, col_ind, values, base, alpha, beta, scalars_on_device, x, y);
    return -1;
}

}  // extern "C"
