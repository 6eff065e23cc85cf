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
#include "spsv_plan.cuh"

namespace b200spsv {

constexpr int      kThreads = 256;                        // solve kernel: 8 warps (rows in flight) per CTA

static void layout(int64_t rows, int64_t nnz, int transpose, size_t* o) {
    size_t p = 0;
    o[B200SPSV_STATE] = p;   p += 256;
    o[B200SPSV_FLAGS] = p;   p += round_up_256(4 * (size_t)rows);
    o[B200SPSV_T_OFF] = p;   p += round_up_256(4 * ((size_t)rows + 1));
    o[B200SPSV_DIAG] = p;    p += round_up_256(4 * (size_t)rows);
    o[B200SPSV_T_COL] = p;   p += round_up_256(4 * (size_t)nnz);
    o[B200SPSV_T_VIDX] = p;  p += round_up_256(4 * (size_t)nnz);
    o[B200SPSV_SCRATCH] = p; p += round_up_256(4 * (size_t)rows) + (transpose ? 2 * round_up_256(4 * (size_t)nnz) : 0);
    o[B200SPSV_TOTAL] = p;
}

// ------------------------------------------------------------------------------------------------ solve
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

template <typename T>
static int launch_solve(cudaStream_t s, int rows, int ascending, int unit, const size_t* o, char* ws, const void* values,
                        const void* diag, const void* alpha, int on_dev, const void* x, void* y) {
    unsigned* state = (unsigned*)(ws + o[B200SPSV_STATE]);
    begin_kernel<<<1, 1, 0, s>>>(state);
    const int cap = resident_ctas<T>(solve_kernel<T>, kThreads);
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
    if (err != cudaSuccess) return (int)err;
    unsigned* state = (unsigned*)(ws + o[B200SPSV_STATE]);
    err = build_plan(s, rows, nnz, (const int*)row_offsets, (const int*)col_ind, base, lower, unit, transpose, state,
                     (int*)(ws + o[B200SPSV_T_OFF]), (int*)(ws + o[B200SPSV_DIAG]), (int*)(ws + o[B200SPSV_T_COL]),
                     (int*)(ws + o[B200SPSV_T_VIDX]), ws + o[B200SPSV_SCRATCH]);
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
