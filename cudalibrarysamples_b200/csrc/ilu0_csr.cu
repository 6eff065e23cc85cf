// ilu0_csr.cu -- incomplete LU and Cholesky factorization without fill-in (cusparse<t>csrilu02 / csric02) for CSR on sm_90a
// (include/b200spmv.h, b200ilu0_*).  DESIGN.md 3.26.
//
// Analysis builds SpSV's plan of the strictly-lower triangle (spsv_plan.cuh): row i depends on the rows k of its entries (i, k),
// k < i, in both factorizations.  It checks the pattern on the device, then computes the level order on the host: order[] lists
// the rows level by level, level_start[] where each level begins.
//
// The factorization is one cooperative launch.  Warps take the rows of a level by static striding, and grid.sync() separates the
// levels: a row reads only its own entries and those of rows of earlier levels, which are final once the barrier is passed.  No
// atomics on values, no flags, no spin waits.  Values are read with ld.global.cg: rows written by other SMs since the launch began
// are never served from a stale L1 line.
//
// One warp per row.  Step k walks the row's strictly-lower entries in ascending column order; lane 0 forms the multiplier, and the
// lanes then update the entries that step touches, each entry by exactly one lane.  Every entry is therefore a left fold in
// ascending k of correctly rounded operations: its bits are the sequential algorithm's (oracle/ilu0_ref.py).
#include <cooperative_groups.h>
#include <cuda_runtime.h>

#include <algorithm>
#include <climits>
#include <cmath>
#include <cstdint>
#include <vector>

#include "../../include/b200spmv.h"
#include "spsv_plan.cuh"

namespace b200ilu0 {

using namespace b200spsv;
namespace cg = cooperative_groups;

constexpr int kThreads = 512;          // 16 warps (rows in flight) per CTA
constexpr int kCtasPerSm = 1;          // a larger grid makes every grid.sync() dearer
// state words after build_plan's four (ST_EPOCH .. ST_MISSING)
enum { W_LEVELS = 4, W_PIVOT = 5, W_PATTERN = 6, W_STRUCT = 7, W_WORDS = 8 };
constexpr unsigned kNone = INT32_MAX;

static void layout(int64_t rows, int64_t nnz, size_t* o) {
    size_t p = 0;
    o[B200ILU0_STATE] = p;       p += 256;
    o[B200ILU0_DIAG] = p;        p += round_up_256(4 * (size_t)rows);
    o[B200ILU0_ORDER] = p;       p += round_up_256(4 * (size_t)rows);
    o[B200ILU0_LEVEL_START] = p; p += round_up_256(4 * ((size_t)rows + 1));
    o[B200ILU0_T_OFF] = p;       p += round_up_256(4 * ((size_t)rows + 1));
    o[B200ILU0_T_COL] = p;       p += round_up_256(4 * (size_t)nnz);
    o[B200ILU0_T_VIDX] = p;      p += round_up_256(4 * (size_t)nnz);
    o[B200ILU0_CHECKED_OFF] = p; p += round_up_256(4 * ((size_t)rows + 1));
    o[B200ILU0_SCRATCH] = p;     p += round_up_256(4 * (size_t)rows);
    o[B200ILU0_TOTAL] = p;
}

__device__ __forceinline__ float sqrt_rn(float a) { return __fsqrt_rn(a); }
__device__ __forceinline__ double sqrt_rn(double a) { return __dsqrt_rn(a); }

static __global__ void init_state_kernel(unsigned* state) {
    state[W_LEVELS] = 0u;
    state[W_PIVOT] = kNone;
    state[W_PATTERN] = 0u;
    state[W_STRUCT] = kNone;
}

// The caller's offsets clamped to [0, nnz] (+ base), so that no analysis kernel indexes col[] outside it; a row whose offsets are
// out of range or decreasing counts as a bad pattern.
static __global__ void offsets_kernel(int rows, int nnz, const int* __restrict__ off, int base, int* __restrict__ checked,
                                      unsigned* state) {
    const int r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r > rows) return;
    const int v = off[r] - base;
    checked[r] = min(max(v, 0), nnz) + base;
    if (v < 0 || v > nnz || (r < rows && off[r + 1] - base < v)) atomicAdd(&state[W_PATTERN], 1u);
}

// Per row of the checked offsets: columns strictly ascending and within [0, rows); the first row without a stored diagonal goes
// to the structural-zero word and, until a factorization runs, to the zero-pivot word.
static __global__ void pattern_kernel(int rows, const int* __restrict__ off, const int* __restrict__ col, int base,
                                      const int* __restrict__ diag, unsigned* state) {
    const int r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= rows) return;
    const int b = off[r] - base, e = off[r + 1] - base;
    bool bad = false;
    int prev = -1;
    for (int k = b; k < e; k++) {
        const int c = col[k] - base;
        if (c <= prev || c >= rows) bad = true;
        prev = c;
    }
    if (bad) atomicAdd(&state[W_PATTERN], 1u);
    if (diag[r] < 0) {
        atomicMin(&state[W_STRUCT], (unsigned)r);
        atomicMin(&state[W_PIVOT], (unsigned)r);
    }
}

// Position of the raw column value c in col[lo, hi) (ascending), or -1.
__device__ __forceinline__ int find_col(const int* __restrict__ col, int lo, int hi, int c) {
    while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        const int v = col[mid];
        if (v == c) return mid;
        if (v < c) lo = mid + 1;
        else hi = mid;
    }
    return -1;
}

// ILU(0), row i (IKJ): for each stored (i, k), k < i ascending: a_ik /= a_kk, then a_ij -= a_ik a_kj for every stored (k, j), j > k,
// that row i also stores.  Then the pivot's boost and zero check.
template <typename T>
__device__ __forceinline__ void ilu_row(int i, int lane, const int* __restrict__ off, const int* __restrict__ col, int base,
                                        const int* __restrict__ diag, T* values, bool boost, double tol, T boost_val, unsigned* state) {
    const int e = off[i + 1] - base, d = diag[i];
    if (d < 0) return;                 // no stored diagonal: the row is left as stored (the structural zero is already reported)
    for (int p = off[i] - base; p < d; p++) {
        const int k = col[p] - base;
        const int dk = diag[k], ek = off[k + 1] - base;
        if (dk < 0) continue;          // nothing is read from a row without a diagonal (warp-uniform)
        T lik = T(0);
        if (lane == 0) {
            lik = div_rn(__ldcg(&values[p]), __ldcg(&values[dk]));
            values[p] = lik;
        }
        lik = __shfl_sync(0xffffffffu, lik, 0);
        for (int q = dk + 1 + lane; q < ek; q += 32) {
            const int pos = find_col(col, p + 1, e, col[q]);
            if (pos >= 0) values[pos] = sub_rn(__ldcg(&values[pos]), mul_rn(lik, __ldcg(&values[q])));
        }
        __syncwarp();                  // this step's updates before the next step's reads
    }
    if (lane == 0) {
        T a = __ldcg(&values[d]);
        if (boost && fabs((double)a) <= tol) {
            a = boost_val;
            values[d] = a;
        }
        if (a == T(0)) atomicMin(&state[W_PIVOT], (unsigned)i);
    }
}

// IC(0), row i, lower triangle only: for each stored (i, k), k < i ascending: l_ik = a_ik / l_kk, a_ij -= l_ik l_jk for every
// stored (i, j), k < j < i, with (j, k) stored, and a_ii -= l_ik l_ik.  Then l_ii = sqrt(a_ii).
template <typename T>
__device__ __forceinline__ void ic_row(int i, int lane, const int* __restrict__ off, const int* __restrict__ col, int base,
                                       const int* __restrict__ diag, T* values, unsigned* state) {
    const int d = diag[i];
    if (d < 0) return;                 // no stored diagonal: the row is left as stored (the structural zero is already reported)
    for (int p = off[i] - base; p < d; p++) {
        const int ck = col[p];
        const int k = ck - base;
        if (diag[k] < 0) continue;     // nothing is read from a row without a diagonal (warp-uniform)
        T lik = T(0);
        if (lane == 0) {
            lik = div_rn(__ldcg(&values[p]), __ldcg(&values[diag[k]]));
            values[p] = lik;
            values[d] = sub_rn(__ldcg(&values[d]), mul_rn(lik, lik));
        }
        lik = __shfl_sync(0xffffffffu, lik, 0);
        for (int q = p + 1 + lane; q < d; q += 32) {
            const int j = col[q] - base;
            const int pos = find_col(col, off[j] - base, diag[j], ck);      // -1 too when row j has no diagonal (diag[j] == -1)
            if (pos >= 0) values[q] = sub_rn(__ldcg(&values[q]), mul_rn(lik, __ldcg(&values[pos])));
        }
        __syncwarp();
    }
    if (lane == 0) {
        const T a = __ldcg(&values[d]);
        if (!(a > T(0))) atomicMin(&state[W_PIVOT], (unsigned)i);
        values[d] = sqrt_rn(a);
    }
}

template <typename T, bool IC>
__global__ void __launch_bounds__(kThreads) ilu0_factor_kernel(const int* __restrict__ off, const int* __restrict__ col, int base,
                                                              const int* __restrict__ diag, const int* __restrict__ order,
                                                              const int* __restrict__ level_start, T* values, int boost,
                                                              const double* tol_dev, double tol_host, const T* boost_dev, T boost_host,
                                                              unsigned* state) {
    cg::grid_group grid = cg::this_grid();
    const int lane = threadIdx.x & 31;
    const int warp = (int)((blockIdx.x * (unsigned)blockDim.x + threadIdx.x) >> 5);
    const int warps = (int)((gridDim.x * (unsigned)blockDim.x) >> 5);
    const int levels = (int)state[W_LEVELS];
    double tol = tol_host;
    T boost_val = boost_host;
    if (boost && tol_dev) tol = *tol_dev;
    if (boost && boost_dev) boost_val = *boost_dev;
    for (int l = 0; l < levels; l++) {
        const int hi = level_start[l + 1];
        for (int q = level_start[l] + warp; q < hi; q += warps) {
            if (IC) ic_row<T>(order[q], lane, off, col, base, diag, values, state);
            else ilu_row<T>(order[q], lane, off, col, base, diag, values, boost != 0, tol, boost_val, state);
        }
        if (l + 1 < levels) grid.sync();
    }
}

static __global__ void zero_pivot_kernel(const unsigned* state, int* position) {
    const unsigned v = state[W_PIVOT];
    *position = v == kNone ? -1 : (int)v;
}

// Resident CTAs of the factorization kernel, capped at kCtasPerSm per SM: the grid of its cooperative launch.
template <typename T, bool IC>
struct FactorTag {};
template <typename T, bool IC>
static int factor_grid() {
    const int cap = resident_ctas<FactorTag<T, IC>>(ilu0_factor_kernel<T, IC>, kThreads);
    int dev = 0, sms = 0;
    if (cap <= 0 || cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess)
        return 0;
    return std::min(cap, sms * kCtasPerSm);
}

template <typename T, bool IC>
static int launch_factor(cudaStream_t s, const size_t* o, char* ws, const int* off, const int* col, int base, void* values, int boost,
                         const void* tol, const void* boost_val, int on_dev) {
    unsigned* state = (unsigned*)(ws + o[B200ILU0_STATE]);
    const int grid = factor_grid<T, IC>();
    if (grid <= 0) return (int)cudaErrorInvalidDevice;
    // the zero-pivot word restarts from the structural zero analysis found
    cudaError_t err = cudaMemcpyAsync(&state[W_PIVOT], &state[W_STRUCT], sizeof(unsigned), cudaMemcpyDeviceToDevice, s);
    if (err != cudaSuccess) return (int)err;
    const int* diag = (const int*)(ws + o[B200ILU0_DIAG]);
    const int* order = (const int*)(ws + o[B200ILU0_ORDER]);
    const int* level_start = (const int*)(ws + o[B200ILU0_LEVEL_START]);
    T* v = (T*)values;
    const bool use = boost && !IC;
    const double* tol_dev = use && on_dev ? (const double*)tol : nullptr;
    double tol_host = use && !on_dev ? *(const double*)tol : 0.0;
    const T* boost_dev = use && on_dev ? (const T*)boost_val : nullptr;
    T boost_host = use && !on_dev ? *(const T*)boost_val : T(0);
    int boost_flag = use ? 1 : 0;
    void* args[] = {(void*)&off, (void*)&col, (void*)&base, (void*)&diag, (void*)&order, (void*)&level_start, (void*)&v, (void*)&boost_flag,
                    (void*)&tol_dev, (void*)&tol_host, (void*)&boost_dev, (void*)&boost_host, (void*)&state};
    return (int)cudaLaunchCooperativeKernel((const void*)ilu0_factor_kernel<T, IC>, dim3(grid), dim3(kThreads), args, 0, s);
}

static bool flag01(int v) { return v == 0 || v == 1; }

}  // namespace b200ilu0

using namespace b200ilu0;

extern "C" {

size_t b200ilu0_workspace_bytes(int64_t rows, int64_t nnz) {
    if (rows < 0 || nnz < 0) return 0;
    size_t o[B200ILU0_LAYOUT_N];
    layout(rows, nnz, o);
    return o[B200ILU0_TOTAL];
}

int b200ilu0_layout(int64_t rows, int64_t nnz, size_t* offsets) {
    if (rows < 0 || nnz < 0 || !offsets) return -1;
    layout(rows, nnz, offsets);
    return 0;
}

void b200ilu0_params(int32_t* threads_per_cta, int32_t* ctas_per_sm) {
    if (threads_per_cta) *threads_per_cta = kThreads;
    if (ctas_per_sm) *ctas_per_sm = kCtasPerSm;
}

int b200ilu0_analysis(void* stream, int64_t rows, int64_t nnz, const void* row_offsets, const void* col_ind, int32_t base, void* workspace,
                      int64_t* structural_zero, int64_t* levels) {
    if (rows < 0 || rows >= INT32_MAX || nnz < 0 || nnz >= INT32_MAX || !flag01(base) || !workspace || ((uintptr_t)workspace & 15) ||
        (rows > 0 && !row_offsets) || (nnz > 0 && !col_ind))
        return -1;
    int dev = 0, coop = 0;
    cudaError_t err = cudaGetDevice(&dev);
    if (err == cudaSuccess) err = cudaDeviceGetAttribute(&coop, cudaDevAttrCooperativeLaunch, dev);
    if (err != cudaSuccess) return (int)err;
    if (!coop) return B200ILU0_NO_COOPERATIVE;
    cudaStream_t s = (cudaStream_t)stream;
    size_t o[B200ILU0_LAYOUT_N];
    layout(rows, nnz, o);
    char* ws = (char*)workspace;
    unsigned* state = (unsigned*)(ws + o[B200ILU0_STATE]);
    int* diag = (int*)(ws + o[B200ILU0_DIAG]);
    int* t_off = (int*)(ws + o[B200ILU0_T_OFF]);
    int* t_col = (int*)(ws + o[B200ILU0_T_COL]);
    int* checked = (int*)(ws + o[B200ILU0_CHECKED_OFF]);
    err = cudaMemsetAsync(state, 0, 256, s);
    if (err != cudaSuccess) return (int)err;
    init_state_kernel<<<1, 1, 0, s>>>(state);
    const int n = (int)rows;
    const int blocks = (n + 1 + kAnalysisThreads - 1) / kAnalysisThreads;
    // Every kernel after this one reads the clamped offsets: a bad offsets array is reported, never followed out of col[].
    offsets_kernel<<<blocks, kAnalysisThreads, 0, s>>>(n, (int)nnz, (const int*)row_offsets, base, checked, state);
    if ((err = cudaGetLastError()) != cudaSuccess) return (int)err;
    err = build_plan(s, rows, nnz, checked, (const int*)col_ind, base, 1, 0, 0, state, t_off, diag, t_col, (int*)(ws + o[B200ILU0_T_VIDX]),
                     ws + o[B200ILU0_SCRATCH]);
    if (err != cudaSuccess) return (int)err;
    if (n > 0) pattern_kernel<<<blocks, kAnalysisThreads, 0, s>>>(n, checked, (const int*)col_ind, base, diag, state);
    if ((err = cudaGetLastError()) != cudaSuccess) return (int)err;
    // The level order is computed on the host from the plan: analysis synchronises once, here (the strictly-lower columns are read
    // back whole, nnz bounding their count), and the factorization never does.
    unsigned words[W_WORDS] = {};
    std::vector<int> h_off(rows + 1, 0), h_col((size_t)nnz), order, level_start;
    err = cudaMemcpyAsync(words, state, sizeof words, cudaMemcpyDeviceToHost, s);
    if (err == cudaSuccess) err = cudaMemcpyAsync(h_off.data(), t_off, 4 * ((size_t)rows + 1), cudaMemcpyDeviceToHost, s);
    if (err == cudaSuccess && nnz > 0) err = cudaMemcpyAsync(h_col.data(), t_col, 4 * (size_t)nnz, cudaMemcpyDeviceToHost, s);
    if (err == cudaSuccess) err = cudaStreamSynchronize(s);
    if (err != cudaSuccess) return (int)err;
    if (words[W_PATTERN] != 0) return B200ILU0_BAD_PATTERN;
    const int64_t nlev = level_order(rows, 1, h_off, h_col, order, &level_start);
    const unsigned nlev_word = (unsigned)nlev;
    // Copies from pageable host memory: each call returns once its source has been staged, so the host arrays may go when it does.
    if (rows > 0) err = cudaMemcpyAsync(ws + o[B200ILU0_ORDER], order.data(), 4 * (size_t)rows, cudaMemcpyHostToDevice, s);
    if (err == cudaSuccess)
        err = cudaMemcpyAsync(ws + o[B200ILU0_LEVEL_START], level_start.data(), 4 * level_start.size(), cudaMemcpyHostToDevice, s);
    if (err == cudaSuccess) err = cudaMemcpyAsync(&state[W_LEVELS], &nlev_word, sizeof nlev_word, cudaMemcpyHostToDevice, s);
    if (err != cudaSuccess) return (int)err;
    if (structural_zero) *structural_zero = words[W_STRUCT] == kNone ? -1 : (int64_t)words[W_STRUCT];
    if (levels) *levels = nlev;
    return 0;
}

int b200ilu0_factor(void* stream, int kind, int dtype, int64_t rows, int64_t nnz, const void* row_offsets, const void* col_ind, int32_t base,
                    void* values, int boost, const void* tol, const void* boost_val, int on_device, void* workspace) {
    if (!flag01(kind) || !flag01(dtype) || rows < 0 || rows >= INT32_MAX || nnz < 0 || nnz >= INT32_MAX || !flag01(base) || !flag01(boost) ||
        !flag01(on_device) || !workspace || ((uintptr_t)workspace & 15) || (rows > 0 && !row_offsets) || (nnz > 0 && (!col_ind || !values)) ||
        (values && ((uintptr_t)values & (dtype ? 7 : 3))) || (boost && kind == B200ILU0_LU && (!tol || !boost_val)))
        return -1;
    if (rows == 0) return 0;
    size_t o[B200ILU0_LAYOUT_N];
    layout(rows, nnz, o);
    cudaStream_t s = (cudaStream_t)stream;
    char* ws = (char*)workspace;
    const int* off = (const int*)row_offsets;
    const int* col = (const int*)col_ind;
    if (kind == B200ILU0_IC)
        return dtype ? launch_factor<double, true>(s, o, ws, off, col, base, values, 0, nullptr, nullptr, on_device)
                     : launch_factor<float, true>(s, o, ws, off, col, base, values, 0, nullptr, nullptr, on_device);
    return dtype ? launch_factor<double, false>(s, o, ws, off, col, base, values, boost, tol, boost_val, on_device)
                 : launch_factor<float, false>(s, o, ws, off, col, base, values, boost, tol, boost_val, on_device);
}

int b200ilu0_zero_pivot(void* stream, const void* workspace, void* position, int on_device, int64_t* row) {
    if (!workspace || ((uintptr_t)workspace & 15) || !position || !flag01(on_device)) return -1;
    cudaStream_t s = (cudaStream_t)stream;
    const unsigned* state = (const unsigned*)workspace;                 // B200ILU0_STATE is at offset 0
    cudaError_t err = cudaSuccess;
    if (on_device) {
        zero_pivot_kernel<<<1, 1, 0, s>>>(state, (int*)position);
        err = cudaGetLastError();
    }
    unsigned v = kNone;
    if (err == cudaSuccess) err = cudaMemcpyAsync(&v, &state[W_PIVOT], sizeof v, cudaMemcpyDeviceToHost, s);
    if (err == cudaSuccess) err = cudaStreamSynchronize(s);
    if (err != cudaSuccess) return (int)err;
    if (!on_device) *(int*)position = v == kNone ? -1 : (int)v;
    if (row) *row = v == kNone ? -1 : (int64_t)v;
    return 0;
}

}  // extern "C"
