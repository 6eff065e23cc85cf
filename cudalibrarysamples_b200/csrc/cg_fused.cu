// cg_fused.cu -- the BLAS-1 part of a CG iteration around the SpMV path, fused and with every scalar kept on the device
// (SURVEY.md 8(f)-2).  Replaces, per iteration of gpu_CG (cuSPARSE/cg/cg_example.c:215-287):
//     cublasDdot(T, P) -> host          (:227)      b200cg_dot           result stays in device memory
//     alpha = delta / denom on the host (:232)      \
//     cublasDaxpy(+alpha, P, X)         (:236-239)   |  b200cg_update_xr   one pass: reads p, t, x, r; writes x, r; r.r
//     cublasDaxpy(-alpha, T, R)         (:241-244)   |                     reduced in the same pass
//     cublasDnrm2(R) -> host            (:247)      /
//     beta = delta_new / delta on host  (:280)      \
//     cublasDscal + cublasDaxpy on P    (:281-286)  /   b200cg_update_p    one pass: p = r + beta * p
// ... or, one vector pass cheaper (10 instead of 11 per iteration, counting every whole-vector read and write including the
// 2 of b200cg_dot: p is read once, next to its own update):
//     b200cg_update_r   r -= alpha t, r.r in the same pass        b200cg_update_xp   x += alpha p_old;  p = r + beta p_old
// No host synchronisation anywhere: scalars are read from / written to device memory, so the whole iteration can be
// captured in a CUDA graph (cuSPARSE/graph_capture/graph_capture_example.c:118-135 shows the pattern for SpVV).
// Reductions are two-level and deterministic: every CTA deposits one partial, the CTA that arrives last adds them in CTA
// order.  fp64 only (the solvers of the reference are fp64: cg_example.c:311, bicgstab_example.c:375).
#include <cuda_runtime.h>
#include <stdint.h>
#include "../../include/b200spmv.h"

namespace b200cg {

constexpr int BLOCK = 256;
constexpr int MAX_CTAS = 132 * 16;   // 256 threads x 16 CTAs/SM candidates: plenty of loads in flight for a pure stream

// workspace: [0 .. MAX_CTAS) partial sums, then one arrival counter (as a double slot)
__device__ __forceinline__ double block_sum(double v, double* sred) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if ((threadIdx.x & 31) == 0) sred[threadIdx.x >> 5] = v;
    __syncthreads();
    double t = 0;
    if (threadIdx.x == 0) {
#pragma unroll
        for (int w = 0; w < BLOCK / 32; w++) t += sred[w];
    }
    return t;      // valid on thread 0
}

// thread 0 of every CTA calls this with its CTA's partial; the last CTA to arrive writes the total (fixed CTA order)
__device__ __forceinline__ void grid_sum_finish(double part, double* ws, double* out) {
    unsigned* counter = (unsigned*)(ws + MAX_CTAS);
    ws[blockIdx.x] = part;
    __threadfence();
    const unsigned arrived = atomicAdd(counter, 1u);
    if (arrived == gridDim.x - 1) {
        __threadfence();
        double t = 0;
        for (unsigned b = 0; b < gridDim.x; b++) t += __ldcg(ws + b);
        *out = t;
        *counter = 0u;
    }
}

__global__ void __launch_bounds__(BLOCK) dot_kernel(int64_t n, const double* __restrict__ a, const double* __restrict__ b,
                                                    double* __restrict__ out, double* __restrict__ ws) {
    __shared__ double sred[BLOCK / 32];
    double s = 0;
    const int64_t stride = (int64_t)gridDim.x * BLOCK * 2;
    for (int64_t i = ((int64_t)blockIdx.x * BLOCK + threadIdx.x) * 2; i < n; i += stride) {
        if (i + 1 < n) {
            const double2 x = *reinterpret_cast<const double2*>(a + i), y = *reinterpret_cast<const double2*>(b + i);
            s += x.x * y.x + x.y * y.y;
        } else {
            s += a[i] * b[i];
        }
    }
    const double t = block_sum(s, sred);
    if (threadIdx.x == 0) grid_sum_finish(t, ws, out);
}

// alpha = delta / denom;  x += alpha p;  r -= alpha t;  delta_new = r . r
__global__ void __launch_bounds__(BLOCK) update_xr_kernel(int64_t n, double* __restrict__ x, double* __restrict__ r,
                                                          const double* __restrict__ p, const double* __restrict__ t,
                                                          const double* __restrict__ delta, const double* __restrict__ denom,
                                                          double* __restrict__ delta_new, double* __restrict__ ws) {
    __shared__ double sred[BLOCK / 32];
    const double alpha = *delta / *denom;
    double s = 0;
    const int64_t stride = (int64_t)gridDim.x * BLOCK * 2;
    for (int64_t i = ((int64_t)blockIdx.x * BLOCK + threadIdx.x) * 2; i < n; i += stride) {
        if (i + 1 < n) {
            const double2 pp = *reinterpret_cast<const double2*>(p + i), tt = *reinterpret_cast<const double2*>(t + i);
            double2 xx = *reinterpret_cast<double2*>(x + i), rr = *reinterpret_cast<double2*>(r + i);
            xx.x += alpha * pp.x; xx.y += alpha * pp.y;
            rr.x -= alpha * tt.x; rr.y -= alpha * tt.y;
            *reinterpret_cast<double2*>(x + i) = xx;
            *reinterpret_cast<double2*>(r + i) = rr;
            s += rr.x * rr.x + rr.y * rr.y;
        } else {
            x[i] += alpha * p[i];
            const double rn = r[i] - alpha * t[i];
            r[i] = rn;
            s += rn * rn;
        }
    }
    const double tt = block_sum(s, sred);
    if (threadIdx.x == 0) grid_sum_finish(tt, ws, delta_new);
}

// beta = delta_new / delta;  p = r + beta p
__global__ void __launch_bounds__(BLOCK) update_p_kernel(int64_t n, double* __restrict__ p, const double* __restrict__ r,
                                                         const double* __restrict__ delta_new, const double* __restrict__ delta) {
    const double beta = *delta_new / *delta;
    const int64_t stride = (int64_t)gridDim.x * BLOCK * 2;
    for (int64_t i = ((int64_t)blockIdx.x * BLOCK + threadIdx.x) * 2; i < n; i += stride) {
        if (i + 1 < n) {
            const double2 rr = *reinterpret_cast<const double2*>(r + i);
            double2 pp = *reinterpret_cast<double2*>(p + i);
            pp.x = rr.x + beta * pp.x; pp.y = rr.y + beta * pp.y;
            *reinterpret_cast<double2*>(p + i) = pp;
        } else {
            p[i] = r[i] + beta * p[i];
        }
    }
}

// --- the same iteration in 10 instead of 11 vector passes (dot included): the x update moves next to the p update (p is read once) ---
// alpha = delta / denom;  r -= alpha t;  delta_new = r . r          (reads t, r; writes r)
__global__ void __launch_bounds__(BLOCK) update_r_kernel(int64_t n, double* __restrict__ r, const double* __restrict__ t,
                                                         const double* __restrict__ delta, const double* __restrict__ denom,
                                                         double* __restrict__ delta_new, double* __restrict__ ws) {
    __shared__ double sred[BLOCK / 32];
    const double alpha = *delta / *denom;
    double s = 0;
    const int64_t stride = (int64_t)gridDim.x * BLOCK * 2;
    for (int64_t i = ((int64_t)blockIdx.x * BLOCK + threadIdx.x) * 2; i < n; i += stride) {
        if (i + 1 < n) {
            const double2 tt = *reinterpret_cast<const double2*>(t + i);
            double2 rr = *reinterpret_cast<double2*>(r + i);
            rr.x -= alpha * tt.x; rr.y -= alpha * tt.y;
            *reinterpret_cast<double2*>(r + i) = rr;
            s += rr.x * rr.x + rr.y * rr.y;
        } else {
            const double rn = r[i] - alpha * t[i];
            r[i] = rn;
            s += rn * rn;
        }
    }
    const double tt = block_sum(s, sred);
    if (threadIdx.x == 0) grid_sum_finish(tt, ws, delta_new);
}

// alpha = delta / denom;  x += alpha p;  beta = delta_new / delta;  p = r + beta p          (reads x, p, r; writes x, p)
__global__ void __launch_bounds__(BLOCK) update_xp_kernel(int64_t n, double* __restrict__ x, double* __restrict__ p,
                                                          const double* __restrict__ r, const double* __restrict__ delta,
                                                          const double* __restrict__ denom, const double* __restrict__ delta_new) {
    const double alpha = *delta / *denom, beta = *delta_new / *delta;
    const int64_t stride = (int64_t)gridDim.x * BLOCK * 2;
    for (int64_t i = ((int64_t)blockIdx.x * BLOCK + threadIdx.x) * 2; i < n; i += stride) {
        if (i + 1 < n) {
            const double2 rr = *reinterpret_cast<const double2*>(r + i);
            double2 pp = *reinterpret_cast<double2*>(p + i), xx = *reinterpret_cast<double2*>(x + i);
            xx.x += alpha * pp.x; xx.y += alpha * pp.y;
            pp.x = rr.x + beta * pp.x; pp.y = rr.y + beta * pp.y;
            *reinterpret_cast<double2*>(x + i) = xx;
            *reinterpret_cast<double2*>(p + i) = pp;
        } else {
            x[i] += alpha * p[i];
            p[i] = r[i] + beta * p[i];
        }
    }
}

static int grid_for(int64_t n) {
    int64_t g = (n / 2 + BLOCK - 1) / BLOCK;
    if (g > MAX_CTAS) g = MAX_CTAS;
    if (g < 1) g = 1;
    return (int)g;
}
static bool aligned16(const void* p) { return ((uintptr_t)p & 15) == 0; }

}  // namespace b200cg

using namespace b200cg;

extern "C" {

size_t b200cg_workspace_bytes(void) { return (MAX_CTAS + 2) * sizeof(double); }

void b200cg_params(int32_t* block, int32_t* max_ctas) {
    if (block) *block = BLOCK;
    if (max_ctas) *max_ctas = MAX_CTAS;
}

// the workspace must be zeroed once (cudaMemset) before its first use; every call leaves the arrival counter at zero
int b200cg_dot(void* stream, int64_t n, const double* a, const double* b, double* out, void* workspace) {
    if (n < 0 || !out || !workspace || (n > 0 && (!a || !b)) || !aligned16(a) || !aligned16(b)) return -1;
    dot_kernel<<<grid_for(n), BLOCK, 0, (cudaStream_t)stream>>>(n, a, b, out, (double*)workspace);
    return (int)cudaGetLastError();
}

int b200cg_update_xr(void* stream, int64_t n, double* x, double* r, const double* p, const double* t, const double* delta,
                     const double* denom, double* delta_new, void* workspace) {
    if (n < 0 || !delta || !denom || !delta_new || !workspace || (n > 0 && (!x || !r || !p || !t))) return -1;
    if (!aligned16(x) || !aligned16(r) || !aligned16(p) || !aligned16(t)) return -1;
    update_xr_kernel<<<grid_for(n), BLOCK, 0, (cudaStream_t)stream>>>(n, x, r, p, t, delta, denom, delta_new, (double*)workspace);
    return (int)cudaGetLastError();
}

int b200cg_update_r(void* stream, int64_t n, double* r, const double* t, const double* delta, const double* denom, double* delta_new,
                    void* workspace) {
    if (n < 0 || !delta || !denom || !delta_new || !workspace || (n > 0 && (!r || !t)) || !aligned16(r) || !aligned16(t)) return -1;
    update_r_kernel<<<grid_for(n), BLOCK, 0, (cudaStream_t)stream>>>(n, r, t, delta, denom, delta_new, (double*)workspace);
    return (int)cudaGetLastError();
}

int b200cg_update_xp(void* stream, int64_t n, double* x, double* p, const double* r, const double* delta, const double* denom,
                     const double* delta_new) {
    if (n < 0 || !delta || !denom || !delta_new || (n > 0 && (!x || !p || !r))) return -1;
    if (!aligned16(x) || !aligned16(p) || !aligned16(r)) return -1;
    update_xp_kernel<<<grid_for(n), BLOCK, 0, (cudaStream_t)stream>>>(n, x, p, r, delta, denom, delta_new);
    return (int)cudaGetLastError();
}

int b200cg_update_p(void* stream, int64_t n, double* p, const double* r, const double* delta_new, const double* delta) {
    if (n < 0 || !delta_new || !delta || (n > 0 && (!p || !r)) || !aligned16(p) || !aligned16(r)) return -1;
    update_p_kernel<<<grid_for(n), BLOCK, 0, (cudaStream_t)stream>>>(n, p, r, delta_new, delta);
    return (int)cudaGetLastError();
}

}  // extern "C"
