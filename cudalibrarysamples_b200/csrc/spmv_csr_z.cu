// spmv_csr_z.cu -- CSR  y = alpha * op(A) * x + beta * y  on H100 (sm_90a) in double complex: A rows x cols CSR with int32 offsets /
// columns (base 0 or 1) and cuDoubleComplex values, x, y, alpha, beta cuDoubleComplex, CUDA_C_64F compute.  Replaces the closed
// library behind cusparseSpMV for a CUDA_C_64F CSR A.  Kept apart from the real-typed CSR kernels (spmv_csr*.cu), which stay as
// they are.
//
// Arithmetic, fixed with intrinsics so that compiler contraction cannot change it (oracle/spmv_csr_z_ref.py restates it):
//   product  a * b      = ( fma(a.re, b.re, -(a.im * b.im)),  fma(a.re, b.im, a.im * b.re) )      (the inner product rounded first)
//   sum      a + b      = ( a.re + b.re,  a.im + b.im )
//   epilogue y_r        = ( fma(al.re, acc.re, fma(-al.im, acc.im, t.re)),  fma(al.re, acc.im, fma(al.im, acc.re, t.im)) ),
//                         t = beta * y_r as a product above; beta == 0 takes t = 0 and never reads y (an empty row gets beta * y).
//
// opA = NON_TRANSPOSE: plan-free and deterministic, the chunked walk of csr_chunk_walk.cuh, with chunks of E = MVZ_CHUNK entries and
// two double2 carry slots per chunk.  A warp streams its chunk's values as 16-byte L1::no_allocate loads and its columns as 4-byte
// ones, one entry per lane per step (coalesced), and gathers x as 16-byte loads through the read-only path.
//
// Shared memory: a product costs 16 bytes, so E = 256 parks 4 KB per warp, 32 KB per 8-warp CTA (+ 4 KB of run sums).  That space
// comes out of the same 256 KB per SM as the L1 that serves the x gather.  The stores are swizzled inside each 8-entry run
// (mvz_swz) so that the lane-per-run summation reads 8 lanes' 16-byte elements from 8 distinct bank groups.  DESIGN.md 3.21 has the
// chunk-size measurement behind E.
//
// opA = TRANSPOSE / CONJUGATE_TRANSPOSE: a scatter shaped like spmv_csr_transpose.cu.  y = beta * y first (beta == 0: zero fill,
// y never read; beta == 1 on the host: skipped), then one warp per 256 entries adds alpha * (v * x[r]) (v conjugated for
// CONJUGATE_TRANSPOSE) to y[c] with two fp64 RED.ADDs per entry.  The order of the additions into a column is not fixed, so results
// agree with a reference to tolerance, not bit for bit (on Gaussian-integer data every sum is exact and they agree bit for bit); the
// closed library makes no reproducibility promise for opA != NON_TRANSPOSE either.
//
// Alignment: y, and values and x when nnz > 0, must be 16-byte aligned (any cuDoubleComplex array is); b200spmv_csr_z rejects
// anything else with -1.
// Nothing past nnz is loaded; x is read only at stored columns.
#include "csr_chunk_walk.cuh"
#include "config.h"
#include "../../include/b200spmv.h"

namespace b200 {

#ifndef B200_CSRZ_CHUNK
#define B200_CSRZ_CHUNK 256         // E: entries per chunk (128 or 256)
#endif
constexpr int MVZ_WARPS = 8;                          // warps (= chunks) per CTA
constexpr int MVZ_CHUNK = B200_CSRZ_CHUNK;
constexpr int MVZ_RUN = 8;                            // R: entries per run
constexpr int MVZ_STEPS = MVZ_CHUNK / 32;             // one entry per lane per step
constexpr int MVZ_RUNS = MVZ_CHUNK / MVZ_RUN;
static_assert(MVZ_CHUNK == 128 || MVZ_CHUNK == 256, "one entry per lane per step, at most 8 steps in registers");
constexpr int MVZ_TR_CHUNK = 256;                     // entries per warp of the transpose scatter

struct SpmvCsrZArgs {
    const int*     off;
    const int*     col;
    const double2* val;
    const double2* x;
    double2*       y;
    double2*       carry;               // split walk: in[c] = carry[2c], out[c] = carry[2c + 1]; nullptr = unsplit
    int            rows, cols, nnz, base, nchunks;
    int            conj;                // transpose scatter: CONJUGATE_TRANSPOSE
};

// Streaming loads that do not allocate in L1.  Not volatile (unlike spmv_common.cuh's): the arrays are read-only for the whole call,
// and a volatile asm pins each load behind the x gather of the step before, which leaves one entry per lane in flight.
__device__ __forceinline__ int mvz_ld_col(const int* p) {
    int r;
    asm("ld.global.nc.L1::no_allocate.s32 %0, [%1];" : "=r"(r) : "l"(p));
    return r;
}
__device__ __forceinline__ double2 mvz_ld_val(const double2* p) {
    double2 r;
    asm("ld.global.nc.L1::no_allocate.v2.f64 {%0,%1}, [%2];" : "=d"(r.x), "=d"(r.y) : "l"(p));
    return r;
}

__device__ __forceinline__ double2 zmul(double2 a, double2 b) {
    return make_double2(__fma_rn(a.x, b.x, -__dmul_rn(a.y, b.y)), __fma_rn(a.x, b.y, __dmul_rn(a.y, b.x)));
}
__device__ __forceinline__ double2 zadd(double2 a, double2 b) { return make_double2(__dadd_rn(a.x, b.x), __dadd_rn(a.y, b.y)); }
__device__ __forceinline__ bool zzero(double2 a) { return a.x == 0.0 && a.y == 0.0; }

// where chunk position p lives in a warp's product array: rotated by its run index inside its run
__device__ __forceinline__ int mvz_swz(int p) { return (p & ~(MVZ_RUN - 1)) | ((p + (p / MVZ_RUN)) & (MVZ_RUN - 1)); }

// Products of chunk c's entries into prod (0 past nnz), then the run sums 0 + p0 + ... + p7 into runs[0 .. E / R).
__device__ __forceinline__ void mvz_products(const SpmvCsrZArgs& a, int c, int lane, double2* prod, double2* runs) {
    const int c0 = c * MVZ_CHUNK;
    int j[MVZ_STEPS];
    double2 v[MVZ_STEPS];
#pragma unroll
    for (int k = 0; k < MVZ_STEPS; k++) {
        const int i = c0 + 32 * k + lane;
        j[k] = a.base;
        v[k] = make_double2(0.0, 0.0);
        if (i < a.nnz) {
            j[k] = mvz_ld_col(a.col + i);
            v[k] = mvz_ld_val(a.val + i);
        }
    }
#pragma unroll
    for (int k = 0; k < MVZ_STEPS; k++) {
        const int p = 32 * k + lane;
        double2 q = make_double2(0.0, 0.0);
        if (c0 + p < a.nnz) q = zmul(v[k], __ldg(a.x + (j[k] - a.base)));
        prod[mvz_swz(p)] = q;
    }
    __syncwarp();
#pragma unroll
    for (int q = lane; q < MVZ_RUNS; q += 32) {
        double2 s = make_double2(0.0, 0.0);
#pragma unroll
        for (int e = 0; e < MVZ_RUN; e++) s = zadd(s, prod[q * MVZ_RUN + ((e + q) & (MVZ_RUN - 1))]);
        runs[q] = s;
    }
    __syncwarp();
}

// y_r = alpha * acc + beta * y_r in the fixed form of the header; beta == 0 never reads y
__device__ __forceinline__ void mvz_store(const SpmvCsrZArgs& a, int r, double2 acc, double2 alpha, double2 beta) {
    const double2 t = zzero(beta) ? make_double2(0.0, 0.0) : zmul(beta, a.y[r]);
    a.y[r] = make_double2(__fma_rn(alpha.x, acc.x, __fma_rn(-alpha.y, acc.y, t.x)), __fma_rn(alpha.x, acc.y, __fma_rn(alpha.y, acc.x, t.y)));
}

// The walk's policy (csr_chunk_walk.cuh): double-complex sums (zadd), products at their swizzled slots
struct MvzWalk {
    using Args = SpmvCsrZArgs;
    using Acc = double2;
    static constexpr int WARPS = MVZ_WARPS, CHUNK = MVZ_CHUNK, RUN = MVZ_RUN;
    static __device__ __forceinline__ double2 zero() { return make_double2(0.0, 0.0); }
    static __device__ __forceinline__ double2 add(double2 u, double2 v) { return zadd(u, v); }
    // v by reference: by value, the chunk kernel compiles to different SASS
    static __device__ __forceinline__ double2 shfl(const double2& v, int src) {
        return make_double2(__shfl_sync(0xffffffffu, v.x, src), __shfl_sync(0xffffffffu, v.y, src));
    }
    static __device__ __forceinline__ int slot(int p) { return mvz_swz(p); }
    static __device__ __forceinline__ void products(const Args& a, int c, int lane, double2* prod, double2* runs) {
        mvz_products(a, c, lane, prod, runs);
    }
    static __device__ __forceinline__ void store(const Args& a, int r, double2 acc, double2 alpha, double2 beta) {
        mvz_store(a, r, acc, alpha, beta);
    }
};

// Two CTAs per SM at least: up to 128 registers, so that all of a lane's column, value and x loads are in flight at once.
__global__ void __launch_bounds__(32 * MVZ_WARPS, 2) spmv_csrz_chunk_kernel(const SpmvCsrZArgs a, const Scalars<double2> sc) {
    __shared__ __align__(16) double2 sprod[MVZ_WARPS][MVZ_CHUNK];
    __shared__ __align__(16) double2 sruns[MVZ_WARPS][MVZ_RUNS];
    csr_walk_chunk<MvzWalk>(a, sc, sprod, sruns);
}

__global__ void __launch_bounds__(CSR_WALK_FIXUP_THREADS) spmv_csrz_fixup_kernel(const SpmvCsrZArgs a, const Scalars<double2> sc) {
    csr_walk_fixup<MvzWalk>(a, sc);
}

// opA = T / C, launch 1: y = beta * y over cols entries (beta == 0: zeros, y never read; beta == 1: nothing to do)
__global__ void spmv_csrz_scale_y_kernel(double2* __restrict__ y, int64_t n, const Scalars<double2> sc) {
    const double2 beta = sc.b();
    if (beta.x == 1.0 && beta.y == 0.0) return;
    const bool zero = zzero(beta);
    // 64-bit index: n may come within one grid stride of 2^31, where i + stride would wrap an int
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
        y[i] = zero ? make_double2(0.0, 0.0) : zmul(beta, y[i]);
}

// opA = T / C, launch 2: every warp owns 256 consecutive entries; entry (r, c, v) adds alpha * (v * x[r]) to y[c] (conj(v) for C)
__global__ void __launch_bounds__(256) spmv_csrz_transpose_kernel(const SpmvCsrZArgs a, const Scalars<double2> sc) {
    const int lane = (int)threadIdx.x & 31;
    const long long wid = (long long)blockIdx.x * 8 + ((int)threadIdx.x >> 5);
    const long long c0 = wid * MVZ_TR_CHUNK;
    if (c0 >= a.nnz) return;                                       // warp-uniform
    const int n0 = (int)c0, n1 = min(n0 + MVZ_TR_CHUNK, a.nnz);
    const double2 alpha = sc.a();
    int r = csr_row_of(a.off, a.rows, a.base, n0);                 // the row of entry n0
    int rend = csr_off(a, r + 1);
    constexpr int STEPS = MVZ_TR_CHUNK / 32;
    int cc[STEPS];
    double2 vv[STEPS];
#pragma unroll
    for (int k = 0; k < STEPS; k++) {
        const int i = n0 + 32 * k + lane;
        cc[k] = a.base;
        vv[k] = make_double2(0.0, 0.0);
        if (i < n1) {
            cc[k] = mvz_ld_col(a.col + i);
            vv[k] = mvz_ld_val(a.val + i);
        }
    }
#pragma unroll
    for (int k = 0; k < STEPS; k++) {
        const int i = n0 + 32 * k + lane;
        if (i < n1) {
            while (rend <= i) { r++; rend = csr_off(a, r + 1); }  // i < nnz = off[rows]: stops at r < rows
            double2 v = vv[k];
            if (a.conj) v.y = -v.y;
            const double2 t = zmul(alpha, zmul(v, __ldg(a.x + r)));
            double2* yc = a.y + (cc[k] - a.base);
            atomicAdd(&yc->x, t.x);
            atomicAdd(&yc->y, t.y);
        }
    }
}

}  // namespace b200

using namespace b200;

extern "C" {

void b200spmv_csr_z_params(int32_t* chunk, int32_t* run, int32_t* warps) {
    if (chunk) *chunk = MVZ_CHUNK;
    if (run) *run = MVZ_RUN;
    if (warps) *warps = MVZ_WARPS;
}

size_t b200spmv_csr_z_workspace_bytes(int64_t rows, int64_t nnz) { return csr_walk_carry_bytes<MVZ_CHUNK, double2>(rows, nnz); }

int b200spmv_csr_z(void* stream, int op, int64_t rows, int64_t cols, int64_t nnz, const void* offsets, const void* columns,
                   const void* values, int32_t base, const void* alpha, const void* beta, int scalars_on_device, const void* x, void* y,
                   void* workspace, size_t workspace_bytes) {
    if (op < 0 || op > 2) return -1;
    if (rows < 0 || cols < 0 || nnz < 0 || !alpha || !beta || (base != 0 && base != 1)) return -1;
    if (rows > INT32_MAX - 64 || cols > INT32_MAX - 64 || nnz > INT32_MAX - 65536) return -1;
    if (nnz > rows * cols) return -1;
    const bool tr = op != 0;
    const int64_t ny = tr ? cols : rows;
    if (ny == 0) return 0;
    if (!y || (rows > 0 && !offsets) || (nnz > 0 && (!columns || !values || !x))) return -1;
    // cuDoubleComplex arrays are 16-byte aligned; values and x are only read when there are entries
    if (((uintptr_t)y & 15) || (nnz > 0 && (((uintptr_t)values | (uintptr_t)x) & 15))) return -1;
    SpmvCsrZArgs a;
    a.off = (const int*)offsets; a.col = (const int*)columns; a.val = (const double2*)values; a.x = (const double2*)x;
    a.y = (double2*)y; a.carry = nullptr;
    a.rows = (int)rows; a.cols = (int)cols; a.nnz = (int)nnz; a.base = base; a.nchunks = (int)csr_walk_nchunks<MVZ_CHUNK>(nnz);
    a.conj = op == 2;
    Scalars<double2> sc;
    set_scalars(sc, alpha, beta, scalars_on_device);
    const cudaStream_t st = (cudaStream_t)stream;
    if (tr) {
        stats().last_csr_kernel = "b200::spmv_csrz_transpose_kernel";
        if (scalars_on_device || !(sc.beta.x == 1.0 && sc.beta.y == 0.0)) {
            int64_t blocks = (cols + 255) / 256;
            if (blocks > 132 * 16) blocks = 132 * 16;
            spmv_csrz_scale_y_kernel<<<(unsigned)blocks, 256, 0, st>>>(a.y, cols, sc);
            const cudaError_t e = cudaGetLastError();
            if (e != cudaSuccess) return (int)e;
        }
        if (nnz == 0 || rows == 0) return 0;
        const int64_t warps = (nnz + MVZ_TR_CHUNK - 1) / MVZ_TR_CHUNK;
        spmv_csrz_transpose_kernel<<<(unsigned)((warps + 7) / 8), 256, 0, st>>>(a, sc);
        return (int)cudaGetLastError();
    }
    a.carry = csr_walk_carry<MVZ_CHUNK, double2>(rows, nnz, workspace, workspace_bytes);
    stats().last_csr_kernel = "b200::spmv_csrz_chunk_kernel";
    return csr_walk_launch<MVZ_WARPS>(st, spmv_csrz_chunk_kernel, spmv_csrz_fixup_kernel, a, sc);
}

}  // extern "C"
