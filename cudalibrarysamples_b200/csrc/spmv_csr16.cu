// spmv_csr16.cu -- CSR  y = alpha * A * x + beta * y  on H100 (sm_90a) in half precision: A rows x cols CSR with int32 offsets /
// columns (base 0 or 1) and fp16 or bf16 values, x of A's type, y of A's type or fp32, fp32 accumulation.  Replaces the closed
// library behind cusparseSpMV for a 16-bit CSR A with fp32 compute.  Kept apart from the fp32 / fp64 CSR kernels (spmv_csr*.cu), which
// stay as they are.
//
// Plan-free and balanced by entries: no preprocess, so the cg / bicgstab call pattern (bufferSize, then SpMV, never preprocess) gets
// the same kernel.  The entry range is cut into chunks of E = MV16_CHUNK entries at fixed positions: chunk c is [c * E, (c + 1) * E).
// One warp takes one chunk:
//   * it finds the chunk's first row with one binary search over the offsets;
//   * it streams the chunk's columns and values, two entries per lane per step (one 64-bit column load and one half2 value load,
//     L1::no_allocate, coalesced: b200spmv_csr16_path), gathers x through the read-only path and parks the fp32 products in shared
//     memory (a 16-bit x 16-bit product is exact in fp32);
//   * a lane sums each run of R = MV16_RUN products (the chunk's entries [8q, 8q + 8)) in order, from 0;
//   * one lane per row then adds the row's piece -- the part of the row inside the chunk -- run by run in ascending order, from 0:
//     a run the piece covers whole contributes its run sum, a run it covers in part contributes 0 + its products in order.
// So the piece sum S(r, c) depends only on the piece's products and its start and end inside the chunk: not on other rows, the grid
// or the SM count.  The row total is acc_r = ((0 + S(r, c0)) + S(r, c0 + 1)) + ..., the pieces in ascending chunk order, and
// y_r = alpha * acc_r + beta * y_r in fp32, rounded once to y's type (beta == 0 never reads y; an empty row gets beta * y).
//
// Split walk (a workspace of b200spmv_csr16_workspace_bytes): a row that starts and ends in one chunk is written by that chunk's warp.
// Each chunk has two fp32 carry slots: in[c] for the piece of the row that enters it from an earlier chunk (at most one), out[c] for
// the piece of the row that starts in c and leaves it (at most one).  spmv_csr16_fixup_kernel owns each such row at its starting
// chunk: it adds out[c], then in[c + 1], in[c + 2], ... and writes y once.  Every slot is written once and read once.
// Unsplit walk (no usable workspace): the warp of a row's starting chunk computes the row's later pieces itself with the same piece
// code and adds them in the same order.  This serialises hub rows, but both walks give identical bits.  No atomics, no allocation,
// no host synchronisation: repeated calls and graph replays give identical bits.
//
// Nothing past nnz is loaded; x is read only at stored columns (a NaN in x[0] reaches exactly the rows that store column 0).
#include "spmv_common.cuh"
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

__device__ __forceinline__ int mv16_off(const SpmvCsr16Args& a, int r) { return __ldg(a.off + r) - a.base; }

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

// S of the piece [s, e) (chunk coordinates): 0 + its runs' sums in ascending order; a run covered in part adds 0 + its products in order
__device__ __forceinline__ float mv16_piece(const float* prod, const float* runs, int s, int e) {
    float acc = 0.f;
    for (int p = s; p < e;) {
        const int q = min(e, (p / MV16_RUN + 1) * MV16_RUN);
        float u;
        if (q - p == MV16_RUN) {
            u = runs[p / MV16_RUN];
        } else {
            u = 0.f;
            for (int i = p; i < q; i++) u = __fadd_rn(u, prod[i]);
        }
        acc = __fadd_rn(acc, u);
        p = q;
    }
    return acc;
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

// One warp per chunk.  Rows handled: the one entering the chunk from an earlier chunk (its piece goes to in[c]) and the rows that
// start in the chunk (the last chunk also takes the empty rows at nnz); of those, the one leaving the chunk goes to out[c].
template <typename T, int LW>
__global__ void __launch_bounds__(32 * MV16_WARPS) spmv_csr16_chunk_kernel(const SpmvCsr16Args a, const Scalars<float> sc) {
    __shared__ __align__(16) float sprod[MV16_WARPS][MV16_CHUNK];
    __shared__ float sruns[MV16_WARPS][MV16_RUNS];
    const int lane = (int)threadIdx.x & 31, warp = (int)threadIdx.x >> 5;
    const int c = (int)blockIdx.x * MV16_WARPS + warp;
    if (c >= a.nchunks) return;
    float* prod = sprod[warp];
    float* runs = sruns[warp];
    const int cs = c * MV16_CHUNK, ce = cs + MV16_CHUNK;
    const bool last = c == a.nchunks - 1;
    // the first row starting at or after cs (off[rows] = nnz >= cs)
    int lo = 0, hi = a.rows;
    while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (mv16_off(a, mid) < cs) lo = mid + 1; else hi = mid;
    }
    mv16_products<T, LW>(a, c, lane, prod, runs);
    const float alpha = sc.a(), beta = sc.b();
    const int r0 = lo > 0 && mv16_off(a, lo) > cs ? lo - 1 : lo;   // the row entering the chunk, if one does
    int leave_row = -1;
    float leave_s = 0.f;
    for (int rb = r0;; rb += 32) {                      // warp-uniform: 32 rows at a time while every lane has one of ours
        const int r = rb + lane;
        int rs = 0, re = 0;
        bool live = r < a.rows;
        if (live) {
            rs = mv16_off(a, r);
            live = last || rs < ce;
        }
        if (live) {
            re = mv16_off(a, r + 1);
            const float s = mv16_piece(prod, runs, max(rs, cs) - cs, min(re, ce) - cs);
            if (rs < cs) {                              // the entering row: the fix-up's (split) or its owner's (unsplit)
                if (a.carry) a.carry[2 * c] = s;
            } else if (re > ce) {                       // the leaving row
                if (a.carry) a.carry[2 * c + 1] = s;
                leave_row = r; leave_s = s;
            } else {
                mv16_store<T>(a, r, __fadd_rn(0.f, s), alpha, beta);
            }
        }
        if (!__all_sync(0xffffffffu, live)) break;
    }
    if (a.carry) return;
    // unsplit: this warp adds the leaving row's later pieces itself, in chunk order, with the same piece code
    const unsigned who = __ballot_sync(0xffffffffu, leave_row >= 0);
    if (!who) return;
    const int src = __ffs(who) - 1;
    const int r = __shfl_sync(0xffffffffu, leave_row, src);
    float acc = __fadd_rn(0.f, __shfl_sync(0xffffffffu, leave_s, src));
    const int re = mv16_off(a, r + 1);
    for (int c2 = c + 1; c2 * MV16_CHUNK < re; c2++) {
        __syncwarp();                                   // every lane is done with the previous chunk's products
        mv16_products<T, LW>(a, c2, lane, prod, runs);
        if (lane == 0) acc = __fadd_rn(acc, mv16_piece(prod, runs, 0, min(re - c2 * MV16_CHUNK, MV16_CHUNK)));
    }
    if (lane == 0) mv16_store<T>(a, r, acc, alpha, beta);
}

// Split walk, part 2: the row that starts in chunk c and leaves it (at most one) gets 0 + out[c] + in[c + 1] + in[c + 2] + ..., in
// ascending chunk order, written once.  One thread per chunk; the last chunk has no such row.
template <typename T>
__global__ void __launch_bounds__(256) spmv_csr16_fixup_kernel(const SpmvCsr16Args a, const Scalars<float> sc) {
    const int c = (int)blockIdx.x * 256 + (int)threadIdx.x;
    if (c >= a.nchunks - 1) return;
    const int cs = c * MV16_CHUNK, ce = cs + MV16_CHUNK;
    const int x = ce - 1;                               // the chunk's last entry (< nnz): the row holding it
    int lo = 0, hi = a.rows;                            // the last r with off[r] <= x
    while (hi - lo > 1) {
        const int mid = (lo + hi) >> 1;
        if (mv16_off(a, mid) <= x) lo = mid; else hi = mid;
    }
    const int rs = mv16_off(a, lo), re = mv16_off(a, lo + 1);
    if (rs < cs || re <= ce) return;                    // it starts before the chunk, or ends in it
    float acc = __fadd_rn(0.f, a.carry[2 * c + 1]);
    for (int c2 = c + 1; c2 * MV16_CHUNK < re; c2++) acc = __fadd_rn(acc, a.carry[2 * c2]);
    mv16_store<T>(a, lo, acc, sc.a(), sc.b());
}

// ------------------------------------------------------------------------------------------------ host side
static int64_t mv16_nchunks(int64_t nnz) { return nnz > 0 ? (nnz + MV16_CHUNK - 1) / MV16_CHUNK : 1; }

static int mv16_path(const void* columns, const void* values) {
    return ((uintptr_t)columns % 8 == 0 && (uintptr_t)values % 4 == 0) ? 2 : 1;
}

template <typename T>
static int launch_mv16(cudaStream_t st, const SpmvCsr16Args& a, const Scalars<float>& sc, int lw) {
    const unsigned ctas = (unsigned)((a.nchunks + MV16_WARPS - 1) / MV16_WARPS);
    if (lw == 2) spmv_csr16_chunk_kernel<T, 2><<<ctas, 32 * MV16_WARPS, 0, st>>>(a, sc);
    else spmv_csr16_chunk_kernel<T, 1><<<ctas, 32 * MV16_WARPS, 0, st>>>(a, sc);
    if (a.carry) spmv_csr16_fixup_kernel<T><<<(unsigned)((a.nchunks - 1 + 255) / 256), 256, 0, st>>>(a, sc);
    return (int)cudaGetLastError();
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

size_t b200spmv_csr16_workspace_bytes(int64_t rows, int64_t nnz) {
    if (rows <= 0 || nnz <= 0) return 0;
    return 2 * (size_t)mv16_nchunks(nnz) * sizeof(float);
}

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
    a.off = (const int*)offsets; a.col = (const int*)columns; a.val = values; a.x = x; a.y = y; a.carry = nullptr;
    a.rows = (int)rows; a.nnz = (int)nnz; a.base = base; a.nchunks = (int)mv16_nchunks(nnz);
    a.y_f32 = y_type == MV16_F32;
    Scalars<float> sc;
    if (scalars_on_device) { sc.alpha = 0.f; sc.beta = 0.f; sc.alpha_dev = (const float*)alpha; sc.beta_dev = (const float*)beta; }
    else { sc.alpha = *(const float*)alpha; sc.beta = *(const float*)beta; sc.alpha_dev = nullptr; sc.beta_dev = nullptr; }
    // the carry slots; a NULL, misaligned or smaller buffer gets the unsplit walk, with the same bits.  One chunk: no row leaves it.
    const size_t need = b200spmv_csr16_workspace_bytes(rows, nnz);
    if (a.nchunks > 1 && workspace && ((uintptr_t)workspace & 15) == 0 && workspace_bytes >= need) a.carry = (float*)workspace;
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
