// spsv_csr.cu -- sparse triangular solve op(T) y = alpha x for CSR on sm_90a (include/b200spsv.h).
//
// Analysis (integer work only) builds the solve plan in the caller's workspace: the selected triangle of op(A) without
// its diagonal, as CSR whose entries point back into the caller's values (t_vidx), plus the diagonal's index per row.
// The solve is sync-free: one warp per row, rows claimed in solve order through an atomic counter, each dependency
// awaited on a per-row ready flag (DESIGN.md section 3.12 has the progress argument).
#include <cuda_runtime.h>

#include <algorithm>
#include <cmath>
#include <cstdint>

#include "../../include/b200spsv.h"

namespace b200spsv {

constexpr int      kThreads = 256;                        // solve kernel: 8 warps (rows in flight) per CTA
constexpr int      kAnalysisThreads = 256;
constexpr int      kScanThreads = 1024;
constexpr uint64_t kSpinBudgetNs = 4000000000ull;         // 4 s per wait: far beyond any legitimate wait, well inside a watchdog
enum { ST_EPOCH = 0, ST_CLAIM = 1, ST_ERROR = 2, ST_MISSING = 3 };

static inline size_t align256(size_t b) { return (b + 255) / 256 * 256; }

static void layout(int64_t rows, int64_t nnz, int transpose, size_t* o) {
    size_t p = 0;
    o[B200SPSV_STATE] = p;   p += 256;
    o[B200SPSV_FLAGS] = p;   p += align256(4 * (size_t)rows);
    o[B200SPSV_T_OFF] = p;   p += align256(4 * ((size_t)rows + 1));
    o[B200SPSV_DIAG] = p;    p += align256(4 * (size_t)rows);
    o[B200SPSV_T_COL] = p;   p += align256(4 * (size_t)nnz);
    o[B200SPSV_T_VIDX] = p;  p += align256(4 * (size_t)nnz);
    o[B200SPSV_SCRATCH] = p; p += align256(4 * (size_t)rows) + (transpose ? 2 * align256(4 * (size_t)nnz) : 0);
    o[B200SPSV_TOTAL] = p;
}

// ------------------------------------------------------------------------------------------------ analysis
// Per row r of A: the first stored diagonal (NON_UNIT), and the number of selected off-diagonal entries -- of row r of
// T (no transpose) or, by atomics, of row c of T^T.  Columns outside [0, rows) are ignored.
__global__ void count_kernel(int rows, const int* __restrict__ off, const int* __restrict__ col, int base, int lower, int unit,
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
__global__ void scan_kernel(int rows, const int* __restrict__ cnt, int* __restrict__ t_off) {
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
__global__ void fill_rows_kernel(int rows, const int* __restrict__ off, const int* __restrict__ col, int base, int lower,
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
__global__ void scatter_cols_kernel(int rows, const int* __restrict__ off, const int* __restrict__ col, int base, int lower,
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
__global__ void order_cols_kernel(int rows, const int* __restrict__ t_off, const int* __restrict__ tmp_row,
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

// ------------------------------------------------------------------------------------------------ solve
__device__ __forceinline__ unsigned ld_acquire(const unsigned* p) {
    unsigned v;
    asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ unsigned ld_relaxed(const unsigned* p) {
    unsigned v;
    asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void st_release(unsigned* p, unsigned v) {
    asm volatile("st.release.gpu.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ uint64_t globaltimer() {
    uint64_t t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    return t;
}

// Waits until row j of this solve is flagged.  false: the budget ran out here (this lane sets the error word) or
// elsewhere in this solve (the error word is already set) -- the caller then writes its row as NaN.
__device__ __forceinline__ bool wait_ready(const unsigned* flag, unsigned epoch, unsigned* err, uint64_t budget) {
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
__global__ void begin_kernel(unsigned* state) {
    state[ST_EPOCH] += 1u;
    state[ST_CLAIM] = 0u;
    state[ST_ERROR] = 0u;
}

template <typename T>
__global__ void __launch_bounds__(kThreads) solve_kernel(int rows, int ascending, int unit, const int* __restrict__ t_off,
                                                         const int* __restrict__ t_col, const int* __restrict__ t_vidx,
                                                         const int* __restrict__ diag_vidx, const T* __restrict__ values,
                                                         const T* __restrict__ diag, const T* __restrict__ alpha_dev, T alpha_host,
                                                         const T* x, T* y, unsigned* flags, unsigned* state, uint64_t budget) {
    const int lane = threadIdx.x & 31;
    const unsigned epoch = ld_relaxed(&state[ST_EPOCH]);     // written by begin_kernel, which ran before this launch
    const T alpha = alpha_dev ? *alpha_dev : alpha_host;
    for (;;) {
        // 1. claim the next row in solve order (a row waits only on rows claimed before it)
        int k = 0;
        if (lane == 0) k = (int)atomicAdd(&state[ST_CLAIM], 1u);
        k = __shfl_sync(0xffffffffu, k, 0);
        if (k >= rows) return;
        const int i = ascending ? k : rows - 1 - k;
        // 2.-3. lanes stride the row's dependencies: wait for each, then read y[j] through L2 (it was written in this launch)
        const int b = t_off[i], e = t_off[i + 1];
        T s = T(0);
        bool bad = false;
        for (int m = b + lane; m < e; m += 32) {
            const int j = t_col[m];
            if (!wait_ready(&flags[j], epoch, &state[ST_ERROR], budget)) bad = true;
            s += values[t_vidx[m]] * __ldcg(&y[j]);
        }
        // 4. fixed shuffle tree: the summation order depends on the plan only
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
        bad = __any_sync(0xffffffffu, bad);
        // 5. the result, then the flag with release semantics
        if (lane == 0) {
            T r = alpha * x[i] - s;
            if (!unit) {
                const int dv = diag_vidx[i];          // -1: no stored diagonal (the shim forwards such matrices)
                r = r / (diag ? diag[i] : (dv >= 0 ? values[dv] : T(NAN)));
            }
            if (bad) r = T(NAN);
            y[i] = r;
            st_release(&flags[i], epoch);
        }
    }
}

// Resident CTAs of solve_kernel<T> on the current device (the persistent grid).  Host queries only: capture-safe.
template <typename T>
static int resident_ctas() {
    static int cache[2][64] = {};
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return 0;
    int& c = cache[sizeof(T) == 8][dev];
    if (c == 0) {
        int sms = 0, per_sm = 0;
        if (cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess ||
            cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, solve_kernel<T>, kThreads, 0) != cudaSuccess)
            return 0;
        c = sms * (per_sm > 0 ? per_sm : 1);
    }
    return c;
}

template <typename T>
static int launch_solve(cudaStream_t s, int rows, int ascending, int unit, const size_t* o, char* ws, const void* values,
                        const void* diag, const void* alpha, int on_dev, const void* x, void* y) {
    unsigned* state = (unsigned*)(ws + o[B200SPSV_STATE]);
    begin_kernel<<<1, 1, 0, s>>>(state);
    const int cap = resident_ctas<T>();
    if (cap <= 0) return (int)cudaErrorInvalidDevice;
    const int warps_per_cta = kThreads / 32;
    const int grid = (int)std::min<int64_t>(cap, ((int64_t)rows + warps_per_cta - 1) / warps_per_cta);
    solve_kernel<T><<<grid, kThreads, 0, s>>>(rows, ascending, unit, (const int*)(ws + o[B200SPSV_T_OFF]),
                                              (const int*)(ws + o[B200SPSV_T_COL]), (const int*)(ws + o[B200SPSV_T_VIDX]),
                                              (const int*)(ws + o[B200SPSV_DIAG]), (const T*)values, (const T*)diag,
                                              on_dev ? (const T*)alpha : nullptr, on_dev ? T(0) : *(const T*)alpha,
                                              (const T*)x, (T*)y, (unsigned*)(ws + o[B200SPSV_FLAGS]), state, kSpinBudgetNs);
    return (int)cudaGetLastError();
}

static bool flag01(int v) { return v == 0 || v == 1; }

}  // namespace b200spsv

using namespace b200spsv;

extern "C" {

size_t b200spsv_csr_workspace_bytes(int64_t rows, int64_t nnz, int transpose) {
    if (rows < 0 || nnz < 0) return 0;
    size_t o[B200SPSV_LAYOUT_N];
    layout(rows, nnz, transpose, o);
    return o[B200SPSV_TOTAL];
}

int b200spsv_csr_layout(int64_t rows, int64_t nnz, int transpose, size_t* offsets) {
    if (rows < 0 || nnz < 0 || !offsets) return -1;
    layout(rows, nnz, transpose, offsets);
    return 0;
}

void b200spsv_csr_params(int32_t* threads_per_cta, uint64_t* spin_budget_ns) {
    if (threads_per_cta) *threads_per_cta = kThreads;
    if (spin_budget_ns) *spin_budget_ns = kSpinBudgetNs;
}

int b200spsv_csr_analysis(void* stream, int64_t rows, int64_t nnz, const void* row_offsets, const void* col_ind, int32_t base,
                          int lower, int unit, int transpose, void* workspace, int64_t* missing_diag) {
    if (rows < 0 || rows >= INT32_MAX || nnz < 0 || nnz >= INT32_MAX || !flag01(base) || !flag01(lower) || !flag01(unit) ||
        !flag01(transpose) || !workspace || ((uintptr_t)workspace & 15) || (rows > 0 && !row_offsets) || (nnz > 0 && !col_ind))
        return -1;
    cudaStream_t s = (cudaStream_t)stream;
    size_t o[B200SPSV_LAYOUT_N];
    layout(rows, nnz, transpose, o);
    char* ws = (char*)workspace;
    cudaError_t err = cudaMemsetAsync(ws, 0, o[B200SPSV_T_OFF], s);                     // state words + ready flags
    if (err == cudaSuccess && rows > 0) err = cudaMemsetAsync(ws + o[B200SPSV_SCRATCH], 0, 4 * (size_t)rows, s);
    if (err != cudaSuccess) return (int)err;
    unsigned* state = (unsigned*)(ws + o[B200SPSV_STATE]);
    int* t_off = (int*)(ws + o[B200SPSV_T_OFF]);
    int* diag = (int*)(ws + o[B200SPSV_DIAG]);
    int* t_col = (int*)(ws + o[B200SPSV_T_COL]);
    int* t_vidx = (int*)(ws + o[B200SPSV_T_VIDX]);
    int* cnt = (int*)(ws + o[B200SPSV_SCRATCH]);
    const int n = (int)rows;
    const int blocks = (n + kAnalysisThreads - 1) / kAnalysisThreads;
    const int* off = (const int*)row_offsets;
    const int* col = (const int*)col_ind;
    if (n > 0) {
        count_kernel<<<blocks, kAnalysisThreads, 0, s>>>(n, off, col, base, lower, unit, transpose, cnt, diag, state);
        scan_kernel<<<1, kScanThreads, 0, s>>>(n, cnt, t_off);
        if (!transpose) {
            fill_rows_kernel<<<blocks, kAnalysisThreads, 0, s>>>(n, off, col, base, lower, t_off, t_col, t_vidx);
        } else {
            int* tmp_row = (int*)(ws + o[B200SPSV_SCRATCH] + align256(4 * (size_t)rows));
            int* tmp_k = (int*)((char*)tmp_row + align256(4 * (size_t)nnz));
            err = cudaMemsetAsync(cnt, 0, 4 * (size_t)rows, s);                                // counts -> cursors
            if (err != cudaSuccess) return (int)err;
            scatter_cols_kernel<<<blocks, kAnalysisThreads, 0, s>>>(n, off, col, base, lower, t_off, cnt, tmp_row, tmp_k);
            const int warps_per_cta = kAnalysisThreads / 32;
            const int oblocks = (int)std::min<int64_t>(65535, ((int64_t)n + warps_per_cta - 1) / warps_per_cta);
            order_cols_kernel<<<oblocks, kAnalysisThreads, 0, s>>>(n, t_off, tmp_row, tmp_k, t_col, t_vidx);
        }
    } else {
        err = cudaMemsetAsync(t_off, 0, 4, s);
        if (err != cudaSuccess) return (int)err;
    }
    err = cudaGetLastError();
    if (err != cudaSuccess) return (int)err;
    if (missing_diag) {
        unsigned m = 0;
        err = cudaMemcpyAsync(&m, &state[ST_MISSING], sizeof m, cudaMemcpyDeviceToHost, s);
        if (err == cudaSuccess) err = cudaStreamSynchronize(s);
        if (err != cudaSuccess) return (int)err;
        *missing_diag = (int64_t)m;
    }
    return 0;
}

int b200spsv_csr_solve(void* stream, int dtype, int64_t rows, int64_t nnz, int lower, int unit, int transpose, const void* values,
                       const void* diag, const void* alpha, int alpha_on_device, const void* x, void* y, void* workspace) {
    if ((dtype != 0 && dtype != 1) || rows < 0 || rows >= INT32_MAX || nnz < 0 || nnz >= INT32_MAX || !flag01(lower) ||
        !flag01(unit) || !flag01(transpose) || !workspace || ((uintptr_t)workspace & 15))
        return -1;
    if (rows == 0) return 0;
    if (!alpha || !x || !y || (nnz > 0 && !values) || (!unit && !values && !diag)) return -1;
    size_t o[B200SPSV_LAYOUT_N];
    layout(rows, nnz, transpose, o);
    const int ascending = lower != transpose;      // effective lower triangle: rows in ascending order
    cudaStream_t s = (cudaStream_t)stream;
    char* ws = (char*)workspace;
    return dtype ? launch_solve<double>(s, (int)rows, ascending, unit, o, ws, values, diag, alpha, alpha_on_device, x, y)
                 : launch_solve<float>(s, (int)rows, ascending, unit, o, ws, values, diag, alpha, alpha_on_device, x, y);
}

}  // extern "C"
