// spsv_plan.cuh -- the triangular-solve plan, its level order and the sync-free wait protocol, shared by spsv_csr.cu
// (libb200spsv.so), spsm_csr.cu and ilu0_csr.cu (libb200spmv.so).  Nothing here is exported: each library gets its own copy.
//
// The plan of op(A)'s selected triangle: t_off / t_col / t_vidx, the triangle without its diagonal as CSR whose entries point
// back into the caller's values, and diag_vidx, the diagonal's index per row (include/b200spsv.h has the layout).
#pragma once

#include <cuda_runtime.h>

#include <algorithm>
#include <cstdint>
#include <vector>

#include "spmv_common.cuh"

namespace b200spsv {

constexpr int      kAnalysisThreads = 256;
constexpr int      kScanThreads = 1024;
constexpr uint64_t kSpinBudgetNs = 4000000000ull;         // 4 s per wait: far beyond any legitimate wait, well inside a watchdog
enum { ST_EPOCH = 0, ST_CLAIM = 1, ST_ERROR = 2, ST_MISSING = 3 };

using b200::round_up_256;

// Correctly rounded operations, never contracted into an FMA: a summation order is then a complete statement of every result's
// bits (oracle/spsm_ref.py and oracle/ilu0_ref.py restate them in numpy).
__device__ __forceinline__ float mul_rn(float a, float b) { return __fmul_rn(a, b); }
__device__ __forceinline__ double mul_rn(double a, double b) { return __dmul_rn(a, b); }
__device__ __forceinline__ float add_rn(float a, float b) { return __fadd_rn(a, b); }
__device__ __forceinline__ double add_rn(double a, double b) { return __dadd_rn(a, b); }
__device__ __forceinline__ float sub_rn(float a, float b) { return __fsub_rn(a, b); }
__device__ __forceinline__ double sub_rn(double a, double b) { return __dsub_rn(a, b); }
__device__ __forceinline__ float div_rn(float a, float b) { return __fdiv_rn(a, b); }
__device__ __forceinline__ double div_rn(double a, double b) { return __ddiv_rn(a, b); }

// ------------------------------------------------------------------------------------------------ analysis
// Per row r of A: the first stored diagonal (NON_UNIT), and the number of selected off-diagonal entries -- of row r of
// T (no transpose) or, by atomics, of row c of T^T.  Columns outside [0, rows) are ignored.
static __global__ void count_kernel(int rows, const int* __restrict__ off, const int* __restrict__ col, int base, int lower, int unit,
                                    int transpose, int* __restrict__ cnt, int* __restrict__ diag_vidx, unsigned* __restrict__ state) {
    const int r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= rows) return;
    const int b = off[r] - base, e = off[r + 1] - base;
    int d = -1, n = 0;
    for (int k = b; k < e; k++) {
        const int c = col[k] - base;
        if (c < 0 || c >= rows) continue;
        if (c == r) {
            if (!unit && d < 0) d = k;
        } else if (lower ? c < r : c > r) {
            if (transpose) atomicAdd(&cnt[c], 1);
            else n++;
        }
    }
    diag_vidx[r] = d;
    if (!transpose) cnt[r] = n;
    if (!unit && d < 0) atomicAdd(&state[ST_MISSING], 1u);
}

// Exclusive scan of cnt[0, rows) into t_off[0, rows], one CTA: each thread sums a contiguous chunk, thread 0 scans the
// chunk sums, each thread writes its chunk.
static __global__ void scan_kernel(int rows, const int* __restrict__ cnt, int* __restrict__ t_off) {
    __shared__ int part[kScanThreads];
    const int64_t chunk = ((int64_t)rows + kScanThreads - 1) / kScanThreads;
    const int64_t lo = min((int64_t)rows, (int64_t)threadIdx.x * chunk), hi = min((int64_t)rows, lo + chunk);
    int s = 0;
    for (int64_t i = lo; i < hi; i++) s += cnt[i];
    part[threadIdx.x] = s;
    __syncthreads();
    if (threadIdx.x == 0) {
        int acc = 0;
        for (int t = 0; t < kScanThreads; t++) { const int v = part[t]; part[t] = acc; acc += v; }
        t_off[rows] = acc;
    }
    __syncthreads();
    int acc = part[threadIdx.x];
    for (int64_t i = lo; i < hi; i++) { t_off[i] = acc; acc += cnt[i]; }
}

// No transpose: row r of T is row r of A's selected triangle, in stored order.
static __global__ void fill_rows_kernel(int rows, const int* __restrict__ off, const int* __restrict__ col, int base, int lower,
                                        const int* __restrict__ t_off, int* __restrict__ t_col, int* __restrict__ t_vidx) {
    const int r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= rows) return;
    const int b = off[r] - base, e = off[r + 1] - base;
    int p = t_off[r];
    for (int k = b; k < e; k++) {
        const int c = col[k] - base;
        if (c < 0 || c >= rows || c == r || (lower ? c > r : c < r)) continue;
        t_col[p] = c;
        t_vidx[p] = k;
        p++;
    }
}

// Transpose, step 1: every selected entry (r, c) lands somewhere in row c of T^T (atomic cursor: order not yet fixed).
static __global__ void scatter_cols_kernel(int rows, const int* __restrict__ off, const int* __restrict__ col, int base, int lower,
                                           const int* __restrict__ t_off, int* __restrict__ cursor, int* __restrict__ tmp_row,
                                           int* __restrict__ tmp_k) {
    const int r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= rows) return;
    const int b = off[r] - base, e = off[r + 1] - base;
    for (int k = b; k < e; k++) {
        const int c = col[k] - base;
        if (c < 0 || c >= rows || c == r || (lower ? c > r : c < r)) continue;
        const int p = t_off[c] + atomicAdd(&cursor[c], 1);
        tmp_row[p] = r;
        tmp_k[p] = k;
    }
}

// Transpose, step 2: one warp per row of T^T puts its entries in ascending stored position (== ascending row of A,
// stored order among duplicates): each entry's rank is the number of smaller positions in the row.  Stable and
// deterministic; the cost is quadratic in the row length, i.e. in the longest column of the triangle.
static __global__ void order_cols_kernel(int rows, const int* __restrict__ t_off, const int* __restrict__ tmp_row,
                                         const int* __restrict__ tmp_k, int* __restrict__ t_col, int* __restrict__ t_vidx) {
    const int lane = threadIdx.x & 31;
    const int warps = gridDim.x * (blockDim.x >> 5);
    for (int c = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); c < rows; c += warps) {
        const int b = t_off[c], n = t_off[c + 1] - b;
        for (int i = lane; i < n; i += 32) {
            const int v = tmp_k[b + i];
            int rank = 0;
            for (int m = 0; m < n; m++) rank += tmp_k[b + m] < v;
            t_vidx[b + rank] = v;
            t_col[b + rank] = tmp_row[b + i];
        }
    }
}

// The launch sequence of the plan, asynchronous on s.  The caller has cleared the state words.  scratch holds cnt[rows]
// (256-byte aligned) and, for transpose, tmp_row[nnz] and tmp_k[nnz] after it, each 256-byte aligned.
static cudaError_t build_plan(cudaStream_t s, int64_t rows, int64_t nnz, const int* off, const int* col, int base, int lower, int unit,
                              int transpose, unsigned* state, int* t_off, int* diag, int* t_col, int* t_vidx, char* scratch) {
    int* cnt = (int*)scratch;
    cudaError_t err = rows > 0 ? cudaMemsetAsync(cnt, 0, 4 * (size_t)rows, s) : cudaSuccess;
    if (err != cudaSuccess) return err;
    const int n = (int)rows;
    const int blocks = (n + kAnalysisThreads - 1) / kAnalysisThreads;
    if (n > 0) {
        count_kernel<<<blocks, kAnalysisThreads, 0, s>>>(n, off, col, base, lower, unit, transpose, cnt, diag, state);
        scan_kernel<<<1, kScanThreads, 0, s>>>(n, cnt, t_off);
        if (!transpose) {
            fill_rows_kernel<<<blocks, kAnalysisThreads, 0, s>>>(n, off, col, base, lower, t_off, t_col, t_vidx);
        } else {
            int* tmp_row = (int*)(scratch + round_up_256(4 * (size_t)rows));
            int* tmp_k = (int*)((char*)tmp_row + round_up_256(4 * (size_t)nnz));
            err = cudaMemsetAsync(cnt, 0, 4 * (size_t)rows, s);                                // counts -> cursors
            if (err != cudaSuccess) return err;
            scatter_cols_kernel<<<blocks, kAnalysisThreads, 0, s>>>(n, off, col, base, lower, t_off, cnt, tmp_row, tmp_k);
            const int warps_per_cta = kAnalysisThreads / 32;
            const int oblocks = (int)std::min<int64_t>(65535, ((int64_t)n + warps_per_cta - 1) / warps_per_cta);
            order_cols_kernel<<<oblocks, kAnalysisThreads, 0, s>>>(n, t_off, tmp_row, tmp_k, t_col, t_vidx);
        }
    } else {
        err = cudaMemsetAsync(t_off, 0, 4, s);
        if (err != cudaSuccess) return err;
    }
    return cudaGetLastError();
}

// Level of every row and the level order, from the plan read back to the host: one pass in the solve direction (every
// dependency of a row precedes it), then a stable counting sort by level.  Returns the number of levels; level_start, when
// not NULL, receives where each level begins in order[] (levels + 1 entries, the last == rows).
static int64_t level_order(int64_t rows, int ascending, const std::vector<int>& t_off, const std::vector<int>& t_col,
                           std::vector<int>& order, std::vector<int>* level_start = nullptr) {
    std::vector<int> level(rows, 0);
    int top = -1;
    for (int64_t k = 0; k < rows; k++) {
        const int64_t i = ascending ? k : rows - 1 - k;
        int l = 0;
        for (int m = t_off[i]; m < t_off[i + 1]; m++) l = std::max(l, level[t_col[m]] + 1);
        level[i] = l;
        top = std::max(top, l);
    }
    std::vector<int64_t> start(top + 2, 0);
    for (int64_t i = 0; i < rows; i++) start[level[i] + 1]++;
    for (int l = 0; l <= top; l++) start[l + 1] += start[l];
    if (level_start) level_start->assign(start.begin(), start.end());
    order.assign(rows, 0);
    for (int64_t k = 0; k < rows; k++) {
        const int64_t i = ascending ? k : rows - 1 - k;
        order[start[level[i]]++] = (int)i;
    }
    return top + 1;
}

// ------------------------------------------------------------------------------------------------ solve protocol
static __device__ __forceinline__ unsigned ld_acquire(const unsigned* p) {
    unsigned v;
    asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
static __device__ __forceinline__ unsigned ld_relaxed(const unsigned* p) {
    unsigned v;
    asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
static __device__ __forceinline__ void st_release(unsigned* p, unsigned v) {
    asm volatile("st.release.gpu.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
static __device__ __forceinline__ uint64_t globaltimer() {
    uint64_t t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    return t;
}

// Waits until row j of this solve is flagged.  false: the budget ran out here (this lane sets the error word) or
// elsewhere in this solve (the error word is already set) -- the caller then writes its row as NaN.
static __device__ __forceinline__ bool wait_ready(const unsigned* flag, unsigned epoch, unsigned* err, uint64_t budget) {
    if (ld_acquire(flag) == epoch) return true;
    const uint64_t t0 = globaltimer();
    for (;;) {
        if (ld_acquire(flag) == epoch) return true;
        if (ld_relaxed(err) != 0) return false;
        if (globaltimer() - t0 > budget) {
            atomicOr(err, 1u);
            return false;
        }
    }
}

// One thread: opens a new solve on this plan (new epoch, no row claimed, no error).
static __global__ void begin_kernel(unsigned* state) {
    state[ST_EPOCH] += 1u;
    state[ST_CLAIM] = 0u;
    state[ST_ERROR] = 0u;
}

// Resident CTAs of a persistent solve kernel on the current device.  Host queries only: capture-safe.  One cache per
// instantiation (Tag tells apart kernels of the same type).
template <typename Tag, typename Kernel>
static int resident_ctas(Kernel kernel, int threads) {
    static int cache[64] = {};
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return 0;
    int& c = cache[dev];
    if (c == 0) {
        int sms = 0, per_sm = 0;
        if (cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess ||
            cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, threads, 0) != cudaSuccess)
            return 0;
        c = sms * (per_sm > 0 ? per_sm : 1);
    }
    return c;
}

}  // namespace b200spsv
