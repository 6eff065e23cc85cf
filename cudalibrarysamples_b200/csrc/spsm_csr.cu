// spsm_csr.cu -- sparse triangular solve with a block of right-hand sides, C = alpha op(T)^-1 op(B), for CSR on sm_90a
// (include/b200spmv.h, b200spsm_*).
//
// Analysis builds SpSV's plan (spsv_plan.cuh) in the caller's workspace, then a level order: a row's level is 1 + the
// largest level among the rows it depends on (0 without dependencies), and order[] lists the rows by (level, position in
// the solve direction).  That is a topological order, so the sync-free protocol of SpSV (DESIGN.md 3.12) keeps its progress
// argument: a claimed row waits only on rows claimed before it.  Claimed in this order, the rows in flight are whole
// levels' worth of independent rows rather than a window of consecutive indices.
//
// The solve is SpSV's persistent claim / flag kernel where each claimed row produces nrhs results (DESIGN.md 3.20 has the
// lane mapping, the memory-ordering argument and the summation order).
#include <cuda_runtime.h>

#include <algorithm>
#include <cmath>
#include <cstdint>
#include <vector>

#include "../../include/b200spmv.h"
#include "spsv_plan.cuh"

namespace b200spsm {

using namespace b200spsv;

constexpr int kThreads = 256;          // solve kernel: 8 warps (rows in flight) per CTA

static void layout(int64_t rows, int64_t nnz, int transpose, size_t* o) {
    size_t p = 0;
    o[B200SPSM_STATE] = p;   p += 256;
    o[B200SPSM_FLAGS] = p;   p += round_up_256(4 * (size_t)rows);
    o[B200SPSM_T_OFF] = p;   p += round_up_256(4 * ((size_t)rows + 1));
    o[B200SPSM_DIAG] = p;    p += round_up_256(4 * (size_t)rows);
    o[B200SPSM_T_COL] = p;   p += round_up_256(4 * (size_t)nnz);
    o[B200SPSM_T_VIDX] = p;  p += round_up_256(4 * (size_t)nnz);
    o[B200SPSM_ORDER] = p;   p += round_up_256(4 * (size_t)rows);
    o[B200SPSM_SCRATCH] = p; p += round_up_256(4 * (size_t)rows) + (transpose ? 2 * round_up_256(4 * (size_t)nnz) : 0);
    o[B200SPSM_TOTAL] = p;
}

// One warp per claimed row.  Lane = g * W + c (W = 1 << tile_log2): c picks a column of the current tile of W right-hand
// sides, g one of 32 / W entry groups; group g sums the row's entries g, g + 32/W, ... in ascending order, and a fixed
// xor tree over the groups adds the partial sums.  op(B)(i, j) = B[i * sbi + j * sbk], C(i, j) = C[i * sci + j * scj].
template <typename T>
__global__ void __launch_bounds__(kThreads) spsm_solve_kernel(int rows, int unit, int tile_log2, int nrhs, const int* __restrict__ order,
                                                              const int* __restrict__ t_off, const int* __restrict__ t_col,
                                                              const int* __restrict__ t_vidx, const int* __restrict__ diag_vidx,
                                                              const T* __restrict__ values, const T* __restrict__ diag,
                                                              const T* __restrict__ alpha_dev, T alpha_host, const T* B, int64_t sbi,
                                                              int64_t sbk, T* C, int64_t sci, int64_t scj, unsigned* flags,
                                                              unsigned* state, uint64_t budget) {
    const int lane = threadIdx.x & 31;
    const int W = 1 << tile_log2, G = 32 >> tile_log2;
    const int c = lane & (W - 1), g = lane >> tile_log2;
    const unsigned epoch = ld_relaxed(&state[ST_EPOCH]);     // written by begin_kernel, which ran before this launch
    const T alpha = alpha_dev ? *alpha_dev : alpha_host;
    for (;;) {
        // 1. claim the next position in level order (a row waits only on rows claimed before it)
        int k = 0;
        if (lane == 0) k = (int)atomicAdd(&state[ST_CLAIM], 1u);
        k = __shfl_sync(0xffffffffu, k, 0);
        if (k >= rows) return;
        const int i = order[k];
        const int b = t_off[i], e = t_off[i + 1];
        // 2. lanes stride the row's dependencies and acquire each flag; the warp barrier then orders every lane's acquire
        //    before every lane's reads of the dependency rows of C
        bool bad = false;
        for (int m = b + lane; m < e; m += 32)
            if (!wait_ready(&flags[t_col[m]], epoch, &state[ST_ERROR], budget)) bad = true;
        __syncwarp();
        bad = __any_sync(0xffffffffu, bad);
        T d = T(1);
        if (!unit) {
            const int dv = diag_vidx[i];              // -1: no stored diagonal (the shim forwards such matrices)
            d = diag ? diag[i] : (dv >= 0 ? values[dv] : T(NAN));
        }
        // 3. tile by tile: per-group partial sums, the xor tree, then lanes of group 0 write their column
        for (int j0 = 0; j0 < nrhs; j0 += W) {
            const int j = j0 + c;
            T s = T(0);
            if (j < nrhs)
                for (int m = b + g; m < e; m += G)
                    s = add_rn(s, mul_rn(values[t_vidx[m]], __ldcg(&C[(int64_t)t_col[m] * sci + (int64_t)j * scj])));
            for (int o = 16; o >= W; o >>= 1) s = add_rn(s, __shfl_xor_sync(0xffffffffu, s, o));
            if (g == 0 && j < nrhs) {
                T r = sub_rn(mul_rn(alpha, B[(int64_t)i * sbi + (int64_t)j * sbk]), s);
                if (!unit) r = div_rn(r, d);
                if (bad) r = T(NAN);
                C[(int64_t)i * sci + (int64_t)j * scj] = r;
            }
        }
        // 4. every lane's writes of row i, then the flag with release semantics (the barrier orders the former before the latter)
        __syncwarp();
        if (lane == 0) st_release(&flags[i], epoch);
    }
}

template <typename T>
static int launch_solve(cudaStream_t s, int rows, int unit, int tile_log2, int nrhs, const size_t* o, char* ws, const void* values,
                        const void* diag, const void* alpha, int on_dev, const void* B, int64_t sbi, int64_t sbk, void* C, int64_t sci,
                        int64_t scj) {
    unsigned* state = (unsigned*)(ws + o[B200SPSM_STATE]);
    begin_kernel<<<1, 1, 0, s>>>(state);
    const int cap = resident_ctas<T>(spsm_solve_kernel<T>, kThreads);
    if (cap <= 0) return (int)cudaErrorInvalidDevice;
    const int warps_per_cta = kThreads / 32;
    const int grid = (int)std::min<int64_t>(cap, ((int64_t)rows + warps_per_cta - 1) / warps_per_cta);
    spsm_solve_kernel<T><<<grid, kThreads, 0, s>>>(
        rows, unit, tile_log2, nrhs, (const int*)(ws + o[B200SPSM_ORDER]), (const int*)(ws + o[B200SPSM_T_OFF]),
        (const int*)(ws + o[B200SPSM_T_COL]), (const int*)(ws + o[B200SPSM_T_VIDX]), (const int*)(ws + o[B200SPSM_DIAG]),
        (const T*)values, (const T*)diag, on_dev ? (const T*)alpha : nullptr, on_dev ? T(0) : *(const T*)alpha, (const T*)B, sbi, sbk,
        (T*)C, sci, scj, (unsigned*)(ws + o[B200SPSM_FLAGS]), state, kSpinBudgetNs);
    return (int)cudaGetLastError();
}

static bool flag01(int v) { return v == 0 || v == 1; }

}  // namespace b200spsm

using namespace b200spsm;

extern "C" {

size_t b200spsm_csr_workspace_bytes(int64_t rows, int64_t nnz, int transpose) {
    if (rows < 0 || nnz < 0) return 0;
    size_t o[B200SPSM_LAYOUT_N];
    layout(rows, nnz, transpose, o);
    return o[B200SPSM_TOTAL];
}

int b200spsm_csr_layout(int64_t rows, int64_t nnz, int transpose, size_t* offsets) {
    if (rows < 0 || nnz < 0 || !offsets) return -1;
    layout(rows, nnz, transpose, offsets);
    return 0;
}

void b200spsm_csr_params(int32_t* threads_per_cta, uint64_t* spin_budget_ns) {
    if (threads_per_cta) *threads_per_cta = kThreads;
    if (spin_budget_ns) *spin_budget_ns = kSpinBudgetNs;
}

int b200spsm_csr_tile(int64_t nrhs, int c_row_major) {
    const int cap = c_row_major ? 32 : 8;
    int w = 1;
    while (w < cap && w < nrhs) w *= 2;
    return w;
}

int b200spsm_csr_analysis(void* stream, int64_t rows, int64_t nnz, const void* row_offsets, const void* col_ind, int32_t base, int lower,
                          int unit, int transpose, void* workspace, int64_t* missing_diag, int64_t* levels) {
    if (rows < 0 || rows >= INT32_MAX || nnz < 0 || nnz >= INT32_MAX || !flag01(base) || !flag01(lower) || !flag01(unit) ||
        !flag01(transpose) || !workspace || ((uintptr_t)workspace & 15) || (rows > 0 && !row_offsets) || (nnz > 0 && !col_ind))
        return -1;
    cudaStream_t s = (cudaStream_t)stream;
    size_t o[B200SPSM_LAYOUT_N];
    layout(rows, nnz, transpose, o);
    char* ws = (char*)workspace;
    cudaError_t err = cudaMemsetAsync(ws, 0, o[B200SPSM_T_OFF], s);                     // state words + ready flags
    if (err != cudaSuccess) return (int)err;
    unsigned* state = (unsigned*)(ws + o[B200SPSM_STATE]);
    int* t_off = (int*)(ws + o[B200SPSM_T_OFF]);
    int* t_col = (int*)(ws + o[B200SPSM_T_COL]);
    err = build_plan(s, rows, nnz, (const int*)row_offsets, (const int*)col_ind, base, lower, unit, transpose, state, t_off,
                     (int*)(ws + o[B200SPSM_DIAG]), t_col, (int*)(ws + o[B200SPSM_T_VIDX]), ws + o[B200SPSM_SCRATCH]);
    if (err != cudaSuccess) return (int)err;
    // The level order is computed on the host from the plan: analysis synchronises here, the solve never does.
    unsigned missing = 0;
    std::vector<int> h_off(rows + 1, 0), h_col, order;
    err = cudaMemcpyAsync(&missing, &state[ST_MISSING], sizeof missing, cudaMemcpyDeviceToHost, s);
    if (err == cudaSuccess) err = cudaMemcpyAsync(h_off.data(), t_off, 4 * ((size_t)rows + 1), cudaMemcpyDeviceToHost, s);
    if (err == cudaSuccess) err = cudaStreamSynchronize(s);
    if (err != cudaSuccess) return (int)err;
    h_col.resize((size_t)h_off[rows]);
    if (!h_col.empty()) err = cudaMemcpyAsync(h_col.data(), t_col, 4 * h_col.size(), cudaMemcpyDeviceToHost, s);
    if (err == cudaSuccess) err = cudaStreamSynchronize(s);
    if (err != cudaSuccess) return (int)err;
    const int64_t nlev = level_order(rows, lower != transpose, h_off, h_col, order);
    if (rows > 0) err = cudaMemcpyAsync(ws + o[B200SPSM_ORDER], order.data(), 4 * (size_t)rows, cudaMemcpyHostToDevice, s);
    if (err == cudaSuccess) err = cudaStreamSynchronize(s);                             // order[] lives on the host until here
    if (err != cudaSuccess) return (int)err;
    if (missing_diag) *missing_diag = (int64_t)missing;
    if (levels) *levels = nlev;
    return 0;
}

int b200spsm_csr_solve(void* stream, int dtype, int64_t rows, int64_t nnz, int unit, const void* values, const void* diag,
                       const void* alpha, int alpha_on_device, int64_t nrhs, const void* B, int64_t sbi, int64_t sbk, void* C,
                       int64_t sci, int64_t scj, void* workspace) {
    if ((dtype != 0 && dtype != 1) || rows < 0 || rows >= INT32_MAX || nnz < 0 || nnz >= INT32_MAX || !flag01(unit) || nrhs < 0 ||
        nrhs > B200SPSM_MAX_NRHS || !workspace || ((uintptr_t)workspace & 15))
        return -1;
    if (rows == 0 || nrhs == 0) return 0;
    if (!alpha || !B || !C || (nnz > 0 && !values) || (!unit && !values && !diag)) return -1;
    size_t o[B200SPSM_LAYOUT_N];
    layout(rows, nnz, 0, o);                                 // every array the solve reads sits before the scratch
    const int w = b200spsm_csr_tile(nrhs, scj == 1);
    int tile_log2 = 0;
    while ((1 << tile_log2) < w) tile_log2++;
    cudaStream_t s = (cudaStream_t)stream;
    char* ws = (char*)workspace;
    return dtype ? launch_solve<double>(s, (int)rows, unit, tile_log2, (int)nrhs, o, ws, values, diag, alpha, alpha_on_device, B, sbi,
                                        sbk, C, sci, scj)
                 : launch_solve<float>(s, (int)rows, unit, tile_log2, (int)nrhs, o, ws, values, diag, alpha, alpha_on_device, B, sbi,
                                       sbk, C, sci, scj);
}

}  // extern "C"
