// cg_reduce.cuh -- the launch shape and the deterministic two-level reduction shared by the fused Krylov BLAS-1 kernels
// (cg_fused.cu, bicgstab_fused.cu).
//
// Every kernel walks its vectors in pairs (16-byte loads, a scalar tail for odd n) with a grid-stride loop over grid_for(n)
// CTAs of BLOCK threads.  A reduction of K values is two-level and fixed in order: each CTA sums its threads (warp shuffles,
// then the warps in order on thread 0) and deposits one partial per value; the CTA that arrives last adds the partials in
// CTA order.  So a result depends on n and the data only, never on timing.
//
// Workspace (doubles): partials of value 0 at [0, MAX_CTAS), the arrival counter (uint32) at slot MAX_CTAS, one spare slot,
// partials of value 1 at [MAX_CTAS + 2, 2 * MAX_CTAS + 2).  A one-value kernel uses the prefix that b200cg_workspace_bytes
// sizes, so one workspace serves both families, and the counter sits at the same byte for every kernel.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include "spmv_common.cuh"

namespace b200cg {

constexpr int BLOCK = 256;
constexpr int MAX_CTAS = 132 * 16;   // 256 threads x 16 CTAs/SM candidates: plenty of loads in flight for a pure stream
constexpr int WS_STRIDE = MAX_CTAS + 2;   // doubles from the partials of one value to those of the next

// v summed over the CTA: the total on thread 0 (0 elsewhere).  sred holds BLOCK / 32 doubles.
__device__ __forceinline__ double block_sum(double v, double* sred) {
    v = b200::warp_allsum(v);
    if ((threadIdx.x & 31) == 0) sred[threadIdx.x >> 5] = v;
    __syncthreads();
    double t = 0;
    if (threadIdx.x == 0) {
#pragma unroll
        for (int w = 0; w < BLOCK / 32; w++) t += sred[w];
    }
    return t;      // valid on thread 0
}

// K values summed over the CTA, in place (valid on thread 0).  sred holds K * BLOCK / 32 doubles; one barrier per value,
// which the one-value kernels' code depends on staying exactly as it is.
template <int K>
__device__ __forceinline__ void block_sum_k(double (&v)[K], double* sred) {
#pragma unroll
    for (int k = 0; k < K; k++) v[k] = block_sum(v[k], sred + k * (BLOCK / 32));
}

// Thread 0 of every CTA calls this with its CTA's K partials.  The last CTA to arrive writes the K totals to out[0 .. K),
// resets the counter and returns true (so it may publish more state that no other CTA of the launch reads); every other
// CTA returns false.
template <int K>
__device__ __forceinline__ bool grid_sum_finish_k(const double (&part)[K], double* ws, double* out) {
    unsigned* counter = (unsigned*)(ws + MAX_CTAS);
#pragma unroll
    for (int k = 0; k < K; k++) ws[k * WS_STRIDE + blockIdx.x] = part[k];
    __threadfence();
    const unsigned arrived = atomicAdd(counter, 1u);
    if (arrived == gridDim.x - 1) {
        __threadfence();
        double t[K];
#pragma unroll
        for (int k = 0; k < K; k++) t[k] = 0;
        for (unsigned b = 0; b < gridDim.x; b++) {
#pragma unroll
            for (int k = 0; k < K; k++) t[k] += __ldcg(ws + k * WS_STRIDE + b);
        }
#pragma unroll
        for (int k = 0; k < K; k++) out[k] = t[k];
        *counter = 0u;
        return true;
    }
    return false;
}

__device__ __forceinline__ void grid_sum_finish(double part, double* ws, double* out) {
    const double a[1] = {part};
    grid_sum_finish_k<1>(a, ws, out);
}

static inline int grid_for(int64_t n) {
    int64_t g = (n / 2 + BLOCK - 1) / BLOCK;
    if (g > MAX_CTAS) g = MAX_CTAS;
    if (g < 1) g = 1;
    return (int)g;
}
static inline bool aligned16(const void* p) { return ((uintptr_t)p & 15) == 0; }

}  // namespace b200cg
