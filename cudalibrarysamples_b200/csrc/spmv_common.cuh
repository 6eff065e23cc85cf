// spmv_common.cuh -- helpers shared by the sparse kernels (sm_90a) and the host code that launches them.
#pragma once
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace b200 {

// ---- streaming loads: val[] / col_ind[] are read exactly once per SpMV, so they bypass L1
//      (ld.global.nc.L1::no_allocate) and leave the whole unified L1 to the gathered x vector. ----
__device__ __forceinline__ int4 ldg_stream_int4(const int* p) {
    int4 r;
    asm volatile("ld.global.nc.L1::no_allocate.v4.s32 {%0,%1,%2,%3}, [%4];"
                 : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p));
    return r;
}
__device__ __forceinline__ int2 ldg_stream_int2(const int* p) {
    int2 r;
    asm volatile("ld.global.nc.L1::no_allocate.v2.s32 {%0,%1}, [%2];" : "=r"(r.x), "=r"(r.y) : "l"(p));
    return r;
}
__device__ __forceinline__ int ldg_stream(const int* p) {
    int r;
    asm volatile("ld.global.nc.L1::no_allocate.s32 %0, [%1];" : "=r"(r) : "l"(p));
    return r;
}
__device__ __forceinline__ double2 ldg_stream_v2(const double* p) {
    double2 r;
    asm volatile("ld.global.nc.L1::no_allocate.v2.f64 {%0,%1}, [%2];" : "=d"(r.x), "=d"(r.y) : "l"(p));
    return r;
}
__device__ __forceinline__ float4 ldg_stream_v4(const float* p) {
    float4 r;
    asm volatile("ld.global.nc.L1::no_allocate.v4.f32 {%0,%1,%2,%3}, [%4];"
                 : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w) : "l"(p));
    return r;
}
__device__ __forceinline__ double ldg_stream(const double* p) {
    double r;
    asm volatile("ld.global.nc.L1::no_allocate.f64 %0, [%1];" : "=d"(r) : "l"(p));
    return r;
}
__device__ __forceinline__ float ldg_stream(const float* p) {
    float r;
    asm volatile("ld.global.nc.L1::no_allocate.f32 %0, [%1];" : "=f"(r) : "l"(p));
    return r;
}

// ---- cold x gathers of csr_flat_kernel with a hot plan: columns outside the packed hot set (spmv_csr_flat.cu).
//      B200_FLAT_COLD picks how they treat L1: 0 = like the hot gather (read-only path, allocating), 1 = L1::evict_first,
//      2 = .cg (L2 only: cold lines never displace the packed hot lines).  2 was fastest on the H100 and 1 slowest
//      (DESIGN.md §3.2, scripts/sweep.py flat_l1).  Not L1::no_allocate: its SASS (LDG.E.NA) is that of the val[] stream. ----
#ifndef B200_FLAT_COLD
#define B200_FLAT_COLD 2
#endif
__device__ __forceinline__ double ldg_cold(const double* p) {
#if B200_FLAT_COLD == 1
    double r;
    asm volatile("ld.global.nc.L1::evict_first.f64 %0, [%1];" : "=d"(r) : "l"(p));
    return r;
#elif B200_FLAT_COLD == 2
    double r;
    asm volatile("ld.global.cg.f64 %0, [%1];" : "=d"(r) : "l"(p));
    return r;
#else
    return __ldg(p);
#endif
}
__device__ __forceinline__ float ldg_cold(const float* p) {
#if B200_FLAT_COLD == 1
    float r;
    asm volatile("ld.global.nc.L1::evict_first.f32 %0, [%1];" : "=f"(r) : "l"(p));
    return r;
#elif B200_FLAT_COLD == 2
    float r;
    asm volatile("ld.global.cg.f32 %0, [%1];" : "=f"(r) : "l"(p));
    return r;
#else
    return __ldg(p);
#endif
}

// 4 consecutive values starting at a 16-byte-aligned element index.
__device__ __forceinline__ void load4_stream(const double* p, double (&v)[4]) {
    double2 a = ldg_stream_v2(p), b = ldg_stream_v2(p + 2);
    v[0] = a.x; v[1] = a.y; v[2] = b.x; v[3] = b.y;
}
__device__ __forceinline__ void load4_stream(const float* p, float (&v)[4]) {
    float4 a = ldg_stream_v4(p);
    v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w;
}

// ---- alpha / beta: by value (CUSPARSE_POINTER_MODE_HOST) or read in-kernel from device memory
//      (CUSPARSE_POINTER_MODE_DEVICE, cusparse.h:275-278). ----
template <typename T>
struct Scalars {
    T        alpha, beta;
    const T* alpha_dev;
    const T* beta_dev;
    __device__ __forceinline__ T a() const { return alpha_dev ? *alpha_dev : alpha; }
    __device__ __forceinline__ T b() const { return beta_dev ? *beta_dev : beta; }
};

// host side: device pointers kept as they are (on_device), host values read now
template <typename T>
void set_scalars(Scalars<T>& s, const void* alpha, const void* beta, int on_device) {
    if (on_device) { s.alpha = T{}; s.beta = T{}; s.alpha_dev = (const T*)alpha; s.beta_dev = (const T*)beta; }
    else { s.alpha = *(const T*)alpha; s.beta = *(const T*)beta; s.alpha_dev = nullptr; s.beta_dev = nullptr; }
}

template <typename T>
__device__ __forceinline__ T axpby(T alpha, T sum, T beta, const T* y) {
    // beta == 0 must not read y (it may hold NaN/uninitialised memory, as cudaMalloc'ed dY does).
    return beta == T(0) ? alpha * sum : alpha * sum + beta * (*y);
}

// B (cols x n, column-major, leading dimension ldb) -> Bt (cols x n, row-major, tight): 32 x 32 tiles through shared memory.
// The row-major copy of a column-major B that spmm_csr.cu (fp32 / fp64) and spmm_csr16.cu (fp16 / bf16) read from the workspace.
// grid.y is capped at 65535 (spmm_transpose_b_grid): a CTA walks the 32-column strips j0, j0 + 32 * gridDim.y, ... so that
// every n up to INT32_MAX - 64 is served, not only n <= 32 * 65535.
template <typename T>
__global__ void __launch_bounds__(256) spmm_transpose_b_kernel(const T* __restrict__ B, long long ldb, T* __restrict__ Bt, int cols, int n) {
    __shared__ T tile[32][33];
    const int tx = (int)threadIdx.x & 31, ty = (int)threadIdx.x >> 5;
    const int k0 = blockIdx.x * 32;
    for (long long j0 = (long long)blockIdx.y * 32; j0 < n; j0 += 32LL * gridDim.y) {      // block-uniform
#pragma unroll
        for (int i = 0; i < 32; i += 8) {
            const int k = k0 + tx;
            const long long j = j0 + ty + i;
            if (k < cols && j < n) tile[ty + i][tx] = B[j * ldb + k];
        }
        __syncthreads();
#pragma unroll
        for (int i = 0; i < 32; i += 8) {
            const int k = k0 + ty + i;
            const long long j = j0 + tx;
            if (k < cols && j < n) Bt[(long long)k * n + j] = tile[tx][ty + i];
        }
        __syncthreads();                                       // the tile is refilled by the next strip
    }
}
inline dim3 spmm_transpose_b_grid(long long cols, long long n) {
    const long long strips = (n + 31) / 32;
    return dim3((unsigned)((cols + 31) / 32), (unsigned)(strips < 65535 ? (strips > 0 ? strips : 1) : 65535));
}

template <typename T>
__device__ __forceinline__ T warp_sum(T v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
    return v;
}

// the warp's sum on every lane (xor butterfly; warp_sum leaves it on lane 0 only)
template <typename T>
__device__ __forceinline__ T warp_allsum(T v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// the row (BSR: block-row) of n holding entry e < nnz: the last r with off[r] - base <= e (an empty row never holds e)
__device__ __forceinline__ int csr_row_of(const int* off, int n, int base, int e) {
    int lo = 0, hi = n;                      // invariant: off[lo] - base <= e < off[hi] - base (off[n] - base = nnz > e)
    while (hi - lo > 1) {
        const int mid = (lo + hi) >> 1;
        if (__ldg(off + mid) - base <= e) lo = mid; else hi = mid;
    }
    return lo;
}

// a stored value widened to its accumulator type: fp16 / bf16 to fp32, fp32 and fp64 as they are
__device__ __forceinline__ float to_acc(__half v) { return __half2float(v); }
__device__ __forceinline__ float to_acc(__nv_bfloat16 v) { return __bfloat162float(v); }
__device__ __forceinline__ float to_acc(float v) { return v; }
__device__ __forceinline__ double to_acc(double v) { return v; }

// workspace sections start on 256-byte boundaries
__host__ __device__ inline size_t round_up_256(size_t b) { return (b + 255) / 256 * 256; }

// the caller's workspace can hold `need` bytes of 16-byte-aligned data
inline bool workspace_usable(const void* ws, size_t bytes, size_t need) {
    return ws && ((uintptr_t)ws & 15) == 0 && bytes >= need;
}

}  // namespace b200
