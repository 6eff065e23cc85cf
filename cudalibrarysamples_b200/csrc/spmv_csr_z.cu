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
// opA = NON_TRANSPOSE: plan-free and deterministic, the walk of spmv_csr16.cu.  No preprocess, so the cg / bicgstab call pattern
// (bufferSize, then SpMV, never preprocess) gets the same kernel.  The entry range is cut into chunks of E = MVZ_CHUNK entries at
// fixed positions; one warp takes one chunk:
//   * it finds the chunk's first row with one binary search over the offsets;
//   * it streams the chunk's values as 16-byte L1::no_allocate loads and its columns as 4-byte ones, one entry per lane per step
//     (coalesced), gathers x as 16-byte loads through the read-only path, and parks the products in shared memory;
//   * a lane sums each run of R = MVZ_RUN products (the chunk's entries [8q, 8q + 8)) in order, from 0;
//   * one lane per row then adds the row's piece -- the part of the row inside the chunk -- run by run in ascending order, from 0:
//     a run the piece covers whole contributes its run sum, a run it covers in part contributes 0 + its products in order.
// The row total is acc_r = ((0 + S(r, c0)) + S(r, c0 + 1)) + ..., its pieces in ascending chunk order.  Split walk (a workspace of
// b200spmv_csr_z_workspace_bytes: two double2 carry slots per chunk) and unsplit walk (no usable workspace) as in spmv_csr16.cu: the
// same pieces in the same order, so both walks, repeated calls and graph replays give identical bits.  No atomics, no allocation.
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
#include "spmv_common.cuh"
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

__device__ __forceinline__ int mvz_off(const SpmvCsrZArgs& a, int r) { return __ldg(a.off + r) - a.base; }

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

// S of the piece [s, e) (chunk coordinates): 0 + its runs' sums in ascending order; a run covered in part adds 0 + its products in order
__device__ __forceinline__ double2 mvz_piece(const double2* prod, const double2* runs, int s, int e) {
    double2 acc = make_double2(0.0, 0.0);
    for (int p = s; p < e;) {
        const int q = min(e, (p / MVZ_RUN + 1) * MVZ_RUN);
        double2 u;
        if (q - p == MVZ_RUN) {
            u = runs[p / MVZ_RUN];
        } else {
            u = make_double2(0.0, 0.0);
            for (int i = p; i < q; i++) u = zadd(u, prod[mvz_swz(i)]);
        }
        acc = zadd(acc, u);
        p = q;
    }
    return acc;
}

// y_r = alpha * acc + beta * y_r in the fixed form of the header; beta == 0 never reads y
__device__ __forceinline__ void mvz_store(const SpmvCsrZArgs& a, int r, double2 acc, double2 alpha, double2 beta) {
    const double2 t = zzero(beta) ? make_double2(0.0, 0.0) : zmul(beta, a.y[r]);
    a.y[r] = make_double2(__fma_rn(alpha.x, acc.x, __fma_rn(-alpha.y, acc.y, t.x)), __fma_rn(alpha.x, acc.y, __fma_rn(alpha.y, acc.x, t.y)));
}

// One warp per chunk.  Rows handled: the one entering the chunk from an earlier chunk (its piece goes to in[c]) and the rows that
// start in the chunk (the last chunk also takes the empty rows at nnz); of those, the one leaving the chunk goes to out[c].
// Two CTAs per SM at least: up to 128 registers, so that all of a lane's column, value and x loads are in flight at once.
__global__ void __launch_bounds__(32 * MVZ_WARPS, 2) spmv_csrz_chunk_kernel(const SpmvCsrZArgs a, const Scalars<double2> sc) {
    __shared__ __align__(16) double2 sprod[MVZ_WARPS][MVZ_CHUNK];
    __shared__ __align__(16) double2 sruns[MVZ_WARPS][MVZ_RUNS];
    const int lane = (int)threadIdx.x & 31, warp = (int)threadIdx.x >> 5;
    const int c = (int)blockIdx.x * MVZ_WARPS + warp;
    if (c >= a.nchunks) return;
    double2* prod = sprod[warp];
    double2* runs = sruns[warp];
    const int cs = c * MVZ_CHUNK, ce = cs + MVZ_CHUNK;
    const bool last = c == a.nchunks - 1;
    // the first row starting at or after cs (off[rows] = nnz >= cs)
    int lo = 0, hi = a.rows;
    while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (mvz_off(a, mid) < cs) lo = mid + 1; else hi = mid;
    }
    mvz_products(a, c, lane, prod, runs);
    const double2 alpha = sc.a(), beta = sc.b();
    const int r0 = lo > 0 && mvz_off(a, lo) > cs ? lo - 1 : lo;     // the row entering the chunk, if one does
    int leave_row = -1;
    double2 leave_s = make_double2(0.0, 0.0);
    for (int rb = r0;; rb += 32) {                      // warp-uniform: 32 rows at a time while every lane has one of ours
        const int r = rb + lane;
        int rs = 0, re = 0;
        bool live = r < a.rows;
        if (live) {
            rs = mvz_off(a, r);
            live = last || rs < ce;
        }
        if (live) {
            re = mvz_off(a, r + 1);
            const double2 s = mvz_piece(prod, runs, max(rs, cs) - cs, min(re, ce) - cs);
            if (rs < cs) {                              // the entering row: the fix-up's (split) or its owner's (unsplit)
                if (a.carry) a.carry[2 * c] = s;
            } else if (re > ce) {                       // the leaving row
                if (a.carry) a.carry[2 * c + 1] = s;
                leave_row = r; leave_s = s;
            } else {
                mvz_store(a, r, zadd(make_double2(0.0, 0.0), s), alpha, beta);
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
    const double2 first = make_double2(__shfl_sync(0xffffffffu, leave_s.x, src), __shfl_sync(0xffffffffu, leave_s.y, src));
    double2 acc = zadd(make_double2(0.0, 0.0), first);
    const int re = mvz_off(a, r + 1);
    for (int c2 = c + 1; c2 * MVZ_CHUNK < re; c2++) {
        __syncwarp();                                   // every lane is done with the previous chunk's products
        mvz_products(a, c2, lane, prod, runs);
        if (lane == 0) acc = zadd(acc, mvz_piece(prod, runs, 0, min(re - c2 * MVZ_CHUNK, MVZ_CHUNK)));
    }
    if (lane == 0) mvz_store(a, r, acc, alpha, beta);
}

// Split walk, part 2: the row that starts in chunk c and leaves it (at most one) gets 0 + out[c] + in[c + 1] + in[c + 2] + ..., in
// ascending chunk order, written once.  One thread per chunk; the last chunk has no such row.
__global__ void __launch_bounds__(256) spmv_csrz_fixup_kernel(const SpmvCsrZArgs a, const Scalars<double2> sc) {
    const int c = (int)blockIdx.x * 256 + (int)threadIdx.x;
    if (c >= a.nchunks - 1) return;
    const int cs = c * MVZ_CHUNK, ce = cs + MVZ_CHUNK;
    const int x = ce - 1;                               // the chunk's last entry (< nnz): the row holding it
    int lo = 0, hi = a.rows;                            // the last r with off[r] <= x
    while (hi - lo > 1) {
        const int mid = (lo + hi) >> 1;
        if (mvz_off(a, mid) <= x) lo = mid; else hi = mid;
    }
    const int rs = mvz_off(a, lo), re = mvz_off(a, lo + 1);
    if (rs < cs || re <= ce) return;                    // it starts before the chunk, or ends in it
    double2 acc = zadd(make_double2(0.0, 0.0), a.carry[2 * c + 1]);
    for (int c2 = c + 1; c2 * MVZ_CHUNK < re; c2++) acc = zadd(acc, a.carry[2 * c2]);
    mvz_store(a, lo, acc, sc.a(), sc.b());
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
    int lo = 0, hi = a.rows;                                       // the row of entry n0: the last r with off[r] <= n0
    while (hi - lo > 1) {
        const int mid = (lo + hi) >> 1;
        if (mvz_off(a, mid) <= n0) lo = mid; else hi = mid;
    }
    int r = lo;
    int rend = mvz_off(a, r + 1);
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
            while (rend <= i) { r++; rend = mvz_off(a, r + 1); }  // i < nnz = off[rows]: stops at r < rows
            double2 v = vv[k];
            if (a.conj) v.y = -v.y;
            const double2 t = zmul(alpha, zmul(v, __ldg(a.x + r)));
            double2* yc = a.y + (cc[k] - a.base);
            atomicAdd(&yc->x, t.x);
            atomicAdd(&yc->y, t.y);
        }
    }
}

// ------------------------------------------------------------------------------------------------ host side
static int64_t mvz_nchunks(int64_t nnz) { return nnz > 0 ? (nnz + MVZ_CHUNK - 1) / MVZ_CHUNK : 1; }

}  // namespace b200

using namespace b200;

extern "C" {

void b200spmv_csr_z_params(int32_t* chunk, int32_t* run, int32_t* warps) {
    if (chunk) *chunk = MVZ_CHUNK;
    if (run) *run = MVZ_RUN;
    if (warps) *warps = MVZ_WARPS;
}

size_t b200spmv_csr_z_workspace_bytes(int64_t rows, int64_t nnz) {
    if (rows <= 0 || nnz <= 0) return 0;
    return 2 * (size_t)mvz_nchunks(nnz) * sizeof(double2);
}

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
    a.rows = (int)rows; a.cols = (int)cols; a.nnz = (int)nnz; a.base = base; a.nchunks = (int)mvz_nchunks(nnz); a.conj = op == 2;
    Scalars<double2> sc;
    if (scalars_on_device) {
        sc.alpha = sc.beta = make_double2(0.0, 0.0);
        sc.alpha_dev = (const double2*)alpha; sc.beta_dev = (const double2*)beta;
    } else {
        sc.alpha = *(const double2*)alpha; sc.beta = *(const double2*)beta; sc.alpha_dev = nullptr; sc.beta_dev = nullptr;
    }
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
    // the carry slots; a NULL, misaligned or smaller buffer gets the unsplit walk, with the same bits.  One chunk: no row leaves it.
    const size_t need = b200spmv_csr_z_workspace_bytes(rows, nnz);
    if (a.nchunks > 1 && workspace && ((uintptr_t)workspace & 15) == 0 && workspace_bytes >= need) a.carry = (double2*)workspace;
    stats().last_csr_kernel = "b200::spmv_csrz_chunk_kernel";
    const unsigned ctas = (unsigned)((a.nchunks + MVZ_WARPS - 1) / MVZ_WARPS);
    spmv_csrz_chunk_kernel<<<ctas, 32 * MVZ_WARPS, 0, st>>>(a, sc);
    if (a.carry) spmv_csrz_fixup_kernel<<<(unsigned)((a.nchunks - 1 + 255) / 256), 256, 0, st>>>(a, sc);
    return (int)cudaGetLastError();
}

}  // extern "C"
