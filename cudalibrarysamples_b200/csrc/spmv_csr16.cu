// spmv_csr16.cu -- CSR  y = alpha * A * x + beta * y  on H100 (sm_90a) in half precision: A rows x cols CSR with int32 offsets /
// columns (base 0 or 1) and fp16 or bf16 values, x of A's type, y of A's type or fp32, fp32 accumulation.  Replaces the closed
// library behind cusparseSpMV for a 16-bit CSR A with fp32 compute.  Kept apart from the fp32 / fp64 CSR kernels (spmv_csr*.cu), which
// stay as they are.
//
// The chunked walk of csr_chunk_walk.cuh, with chunks of E = MV16_CHUNK entries and two fp32 carry slots per chunk.  What is this
// file's own: a warp streams its chunk two entries per lane per step (one 64-bit column load and one half2 value load,
// L1::no_allocate, coalesced: b200spmv_csr16_path), gathers x through the read-only path and parks the fp32 products in shared memory
// (a 16-bit x 16-bit product is exact in fp32); every sum is a __fadd_rn; y_r = alpha * acc_r + beta * y_r in fp32, rounded once to
// y's type.  A NaN in x[0] reaches exactly the rows that store column 0.
#include "csr_chunk_walk.cuh"
#include "config.h"
#include "../../include/b200spmv.h"

#include <cuda_bf16.h>
#include <cuda_fp16.h>

namespace b200 {

#ifndef B200_CSR16_CHUNK
#define B200_CSR16_CHUNK 256        // E: entries per chunk (a multiple of 256)
#endif
constexpr int MV16_WARPS = 8;                         // warps (= chunks) per CTA
constexpr int MV16_CHUNK = B200_CSR16_CHUNK;
constexpr int MV16_RUN = 8;                           // R: entries per run
constexpr int MV16_STEPS = MV16_CHUNK / 64;           // two entries per lane per step
constexpr int MV16_RUNS = MV16_CHUNK / MV16_RUN;
static_assert(MV16_CHUNK % 256 == 0, "a chunk is a whole number of 32-lane run rounds");
constexpr int MV16_F32 = 0, MV16_F16 = 2, MV16_BF16 = 14;   // cudaDataType values

struct SpmvCsr16Args {
    const int* off;
    const int* col;
    const void* val;
    const void* x;
    void*       y;
    float*      carry;                  // split walk: in[c] = carry[2c], out[c] = carry[2c + 1]; nullptr = unsplit
    int         rows, nnz, base, nchunks;
    int         y_f32;                  // y is fp32 (else A's type)
};

__device__ __forceinline__ unsigned ldg_stream_u32(const void* p) {
    unsigned r;
    asm volatile("ld.global.nc.L1::no_allocate.b32 %0, [%1];" : "=r"(r) : "l"(p));
    return r;
}
__device__ __forceinline__ unsigned short ldg_stream_u16(const void* p) {
    unsigned short r;
    asm volatile("ld.global.nc.L1::no_allocate.b16 %0, [%1];" : "=h"(r) : "l"(p));
    return r;
}

// the 16-bit pattern b of A's type as fp32 (exact)
template <typename T>
__device__ __forceinline__ float mv16_f(unsigned short b) {
    if constexpr (std::is_same<T, __half>::value) return __half2float(__ushort_as_half(b));
    else return __uint_as_float((unsigned)b << 16);
}

// Products of chunk c's entries into prod[0 .. E) (0 past nnz), then the run sums 0 + p0 + ... + p7 into runs[0 .. E / R).
// LW = 2: one 64-bit column load and one 32-bit value load per lane per step; LW = 1: scalar loads (a misaligned view).
template <typename T, int LW>
__device__ __forceinline__ void mv16_products(const SpmvCsr16Args& a, int c, int lane, float* prod, float* runs) {
    const int c0 = c * MV16_CHUNK;
    const unsigned short* vals = (const unsigned short*)a.val;
    const unsigned short* xs = (const unsigned short*)a.x;
    int j0[MV16_STEPS], j1[MV16_STEPS];
    unsigned v[MV16_STEPS];
#pragma unroll
    for (int k = 0; k < MV16_STEPS; k++) {
        const int i = c0 + 64 * k + 2 * lane;
        j0[k] = j1[k] = 0;
        v[k] = 0;
        if (LW == 2 && i + 1 < a.nnz) {
            const int2 cc = ldg_stream_int2(a.col + i);
            j0[k] = cc.x; j1[k] = cc.y;
            v[k] = ldg_stream_u32(vals + i);
        } else {
            if (i < a.nnz) { j0[k] = ldg_stream(a.col + i); v[k] = ldg_stream_u16(vals + i); }
            if (i + 1 < a.nnz) { j1[k] = ldg_stream(a.col + i + 1); v[k] |= (unsigned)ldg_stream_u16(vals + i + 1) << 16; }
        }
    }
#pragma unroll
    for (int k = 0; k < MV16_STEPS; k++) {
        const int i = c0 + 64 * k + 2 * lane;
        float2 p = make_float2(0.f, 0.f);
        if (i < a.nnz) p.x = __fmul_rn(mv16_f<T>((unsigned short)v[k]), mv16_f<T>(__ldg(xs + (j0[k] - a.base))));
        if (i + 1 < a.nnz) p.y = __fmul_rn(mv16_f<T>((unsigned short)(v[k] >> 16)), mv16_f<T>(__ldg(xs + (j1[k] - a.base))));
        *(float2*)(prod + 64 * k + 2 * lane) = p;
    }
    __syncwarp();
#pragma unroll
    for (int q = lane; q < MV16_RUNS; q += 32) {
        const float4 lo = *(const float4*)(prod + q * MV16_RUN), hi = *(const float4*)(prod + q * MV16_RUN + 4);
        float s = __fadd_rn(0.f, lo.x);
        s = __fadd_rn(s, lo.y); s = __fadd_rn(s, lo.z); s = __fadd_rn(s, lo.w);
        s = __fadd_rn(s, hi.x); s = __fadd_rn(s, hi.y); s = __fadd_rn(s, hi.z); s = __fadd_rn(s, hi.w);
        runs[q] = s;
    }
    __syncwarp();
}

// y_r = alpha * acc + beta * y_r in fp32, rounded once to y's type; beta == 0 never reads y
template <typename T>
__device__ __forceinline__ void mv16_store(const SpmvCsr16Args& a, int r, float acc, float alpha, float beta) {
    if (a.y_f32) {
        float* p = (float*)a.y + r;
        *p = beta == 0.f ? __fmul_rn(alpha, acc) : __fmaf_rn(alpha, acc, __fmul_rn(beta, *p));
    } else {
        T* p = (T*)a.y + r;
        float yv = 0.f;
        if (beta != 0.f) {
            if constexpr (std::is_same<T, __half>::value) yv = __half2float(*p);
            else yv = __bfloat162float(*p);
        }
        const float v = beta == 0.f ? __fmul_rn(alpha, acc) : __fmaf_rn(alpha, acc, __fmul_rn(beta, yv));
        if constexpr (std::is_same<T, __half>::value) *p = __float2half_rn(v);
        else *p = __float2bfloat16_rn(v);
    }
}

// The walk's policy (csr_chunk_walk.cuh) for A of type T, with LW as in mv16_products: fp32 sums, products in place.  The fix-up
// reads no products, so the LW it is given does not matter.
template <typename T, int LW>
struct Mv16Walk {
    using Args = SpmvCsr16Args;
    using Acc = float;
    static constexpr int WARPS = MV16_WARPS, CHUNK = MV16_CHUNK, RUN = MV16_RUN;
    static __device__ __forceinline__ float zero() { return 0.f; }
    static __device__ __forceinline__ float add(float u, float v) { return __fadd_rn(u, v); }
    static __device__ __forceinline__ float shfl(float v, int src) { return __shfl_sync(0xffffffffu, v, src); }
    static __device__ __forceinline__ int slot(int p) { return p; }
    static __device__ __forceinline__ void products(const Args& a, int c, int lane, float* prod, float* runs) {
        mv16_products<T, LW>(a, c, lane, prod, runs);
    }
    static __device__ __forceinline__ void store(const Args& a, int r, float acc, float alpha, float beta) {
        mv16_store<T>(a, r, acc, alpha, beta);
    }
};

template <typename T, int LW>
__global__ void __launch_bounds__(32 * MV16_WARPS) spmv_csr16_chunk_kernel(const SpmvCsr16Args a, const Scalars<float> sc) {
    __shared__ __align__(16) float sprod[MV16_WARPS][MV16_CHUNK];
    __shared__ float sruns[MV16_WARPS][MV16_RUNS];
    csr_walk_chunk<Mv16Walk<T, LW>>(a, sc, sprod, sruns);
}

template <typename T>
__global__ void __launch_bounds__(CSR_WALK_FIXUP_THREADS) spmv_csr16_fixup_kernel(const SpmvCsr16Args a, const Scalars<float> sc) {
    csr_walk_fixup<Mv16Walk<T, 2>>(a, sc);
}

// ------------------------------------------------------------------------------------------------ host side
static int mv16_path(const void* columns, const void* values) {
    return ((uintptr_t)columns % 8 == 0 && (uintptr_t)values % 4 == 0) ? 2 : 1;
}

template <typename T>
static int launch_mv16(cudaStream_t st, const SpmvCsr16Args& a, const Scalars<float>& sc, int lw) {
    return csr_walk_launch<MV16_WARPS>(st, lw == 2 ? spmv_csr16_chunk_kernel<T, 2> : spmv_csr16_chunk_kernel<T, 1>,
                                       spmv_csr16_fixup_kernel<T>, a, sc);
}

}  // namespace b200

using namespace b200;

extern "C" {

void b200spmv_csr16_params(int32_t* chunk, int32_t* run, int32_t* warps) {
    if (chunk) *chunk = MV16_CHUNK;
    if (run) *run = MV16_RUN;
    if (warps) *warps = MV16_WARPS;
}

int b200spmv_csr16_path(const void* columns, const void* values) { return mv16_path(columns, values); }

size_t b200spmv_csr16_workspace_bytes(int64_t rows, int64_t nnz) { return csr_walk_carry_bytes<MV16_CHUNK, float>(rows, nnz); }

int b200spmv_csr16(void* stream, int a_type, int y_type, int64_t rows, int64_t cols, int64_t nnz, const void* offsets,
                   const void* columns, const void* values, int32_t base, const void* alpha, const void* beta, int scalars_on_device,
                   const void* x, void* y, void* workspace, size_t workspace_bytes) {
    if (a_type != MV16_F16 && a_type != MV16_BF16) return -1;
    if (y_type != a_type && y_type != MV16_F32) return -1;
    if (rows < 0 || cols < 0 || nnz < 0 || !alpha || !beta || (base != 0 && base != 1)) return -1;
    if (rows > INT32_MAX - 64 || cols > INT32_MAX - 64 || nnz > INT32_MAX - 65536) return -1;
    if (nnz > rows * cols) return -1;
    if (rows == 0) return 0;
    if (!y || !offsets || (nnz > 0 && (!columns || !values || !x))) return -1;
    SpmvCsr16Args a;
    a.off = (const int*)offsets; a.col = (const int*)columns; a.val = values; a.x = x; a.y = y;
    a.carry = csr_walk_carry<MV16_CHUNK, float>(rows, nnz, workspace, workspace_bytes);
    a.rows = (int)rows; a.nnz = (int)nnz; a.base = base; a.nchunks = (int)csr_walk_nchunks<MV16_CHUNK>(nnz);
    a.y_f32 = y_type == MV16_F32;
    Scalars<float> sc;
    set_scalars(sc, alpha, beta, scalars_on_device);
    const int lw = mv16_path(columns, values);
    const cudaStream_t st = (cudaStream_t)stream;
    if (a_type == MV16_F16) {
        stats().last_csr_kernel = "b200::spmv_csr16_chunk_kernel<__half>";
        return launch_mv16<__half>(st, a, sc, lw);
    }
    stats().last_csr_kernel = "b200::spmv_csr16_chunk_kernel<__nv_bfloat16>";
    return launch_mv16<__nv_bfloat16>(st, a, sc, lw);
}

}  // extern "C"
