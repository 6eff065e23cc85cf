// spmm_bsr.cu -- BSR x dense  C = alpha * A * op(B) + beta * C  on H100 (sm_90a): A m x k in square bs x bs blocks (int32 block
// offsets / block columns, base 0 or 1, each block stored row- or column-major), op(B) k x n and C m x n dense.  Replaces the closed
// library behind cusparseSpMM for BSR descriptors: the P . V of block-sparse attention, on the pattern whose Q . K^T sddmm_bsr.cu
// computes.  op(B) is reduced to element strides as in sddmm_bsr.cu: op(B)(k, j) = B[k * sbk + j * sbj].
//
//   * Tensor path (fp16 / bf16 A and B, C of that type or fp32, bs % 16 == 0, row-major blocks, 16-byte aligned values and B, op(B)
//     contiguous along K or N with the other stride a multiple of 8): spmm_bsr_mma_kernel.  A CTA of 4 warps owns BM rows of one block-row (BM = 64,
//     32 or 16, the largest that divides bs) and BN = 64 or 128 columns of C (128 whenever n > 64, so an attention head of 128 reads
//     each A block once).  A stored block is contiguous: its BM x 16 slabs and the 16 x BN slices of B its block column selects
//     stream through a SPMM_BSR_STAGES-deep cp.async pipeline, SPMM_BSR_SLABS slabs per stage, so one barrier covers 64 of K at
//     every bs (four bs-16 blocks, two bs-32 blocks, or 64 of one wider block).  ldmatrix (.trans for an N-contiguous B) feeds mma.sync.m16n8k16 with fp32 accumulators.  About n flop per byte of A: bound by streaming A.
//   * CUDA-core path (fp32 on FFMA, fp64 on DFMA, no TF32; every bs; every 16-bit call the tensor path cannot take, column-major
//     blocks among them):
//     spmm_bsr_fma_kernel, a CTA of 32 x 8 threads owning 32 rows of one block-row x 32 columns, each thread 4 rows of one column.
//
// Balance.  A global block-row of the window-plus-global attention pattern stores every block column: one CTA per block-row would
// serialise the layer on it, and one CTA per block-row is too few CTAs to keep HBM busy at sequence length 16384 and bs 64.  Block-rows
// are cut into pieces of at most `ch` stored blocks: ch = max(SPMM_BSR_CHUNK_MIN, min(ceil(SPMM_BSR_CHUNK_FACTOR * bnnz / block-rows),
// ceil(bnnz * batch * ceil(bs / 64) * ceil(n / 128) / SPMM_BSR_TARGET_CTAS))), a function of the shape alone.  With a workspace (the split
// walk) CTA c takes the pieces that start in stored blocks [c * ch, (c + 1) * ch): at most 2 ch blocks.  A block-row of one piece is
// written to C at once; the pieces of a longer row go to carry slots (at most two per chunk: the piece of a row that began in an
// earlier chunk, and the first piece of a long row), and spmm_bsr_fixup_kernel adds them in ascending order and writes the row, and
// writes beta * C for block-rows that store nothing.  Without a usable workspace (the unsplit walk) one CTA walks one block-row and
// adds its pieces in the same order in registers: both walks give the same bits.
// Every C entry is written exactly once, in a fixed order, without atomics: repeated calls and graph replays give identical bits.
// beta == 0 never reads C.  Nothing past n, in ld padding, or in a row of op(B) no stored block references is read.  A strided batch
// is one launch (blockIdx.z).  No allocation, no host synchronisation.
#include "mma_sm90.cuh"
#include "spmv_common.cuh"
#include "../../include/b200spmv.h"

#include <algorithm>
#include <cmath>

namespace b200 {

constexpr int SPMM_BSR_KS = 16;            // K of one slab = K of one mma (tensor path)
constexpr int SPMM_BSR_SLABS = 4;          // slabs per pipeline stage: 64 of K per barrier
constexpr int SPMM_BSR_STAGES = 3;         // stages in flight
constexpr int SPMM_BSR_THREADS = 128;      // tensor path: 4 warps
constexpr int SPMM_BSR_MAX_BM = 64;        // rows of one block-row a tensor-path CTA owns at most
constexpr int SPMM_BSR_PAD = 8;            // halves of row padding in shared memory: ldmatrix rows land in distinct banks
constexpr int SPMM_BSR_CHUNK_MIN = 2;      // stored blocks per piece / chunk: at least this, at most this many times the average
constexpr int SPMM_BSR_CHUNK_FACTOR = 2;   //   block-row, and within those bounds as many as make about SPMM_BSR_TARGET_CTAS CTAs
constexpr int SPMM_BSR_TARGET_CTAS = 1024; //   (counting one CTA per 64 rows of a block and 128 columns of C, per batch matrix)
constexpr int SPMM_BSR_FX = 32, SPMM_BSR_FY = 8, SPMM_BSR_FMR = 4;   // CUDA-core path: 32 columns x (8 x 4) rows per CTA
constexpr int SPMM_BSR_FIX_M = 32, SPMM_BSR_FIX_N = 64;              // fix-up tile

constexpr int MM_F32 = 0, MM_F64 = 1, MM_F16 = 2, MM_BF16 = 14;   // cudaDataType values

struct SpmmBsrArgs {
    const int* off;
    const int* col;
    const void* val;
    const void* B;
    void*       C;
    void*       carry;                  // split walk: [batch][2 * nchunks][bs][n] partial sums (fp32, fp64 for fp64); nullptr = unsplit
    long long   sbk, sbj, ldc;          // op(B)(k, j) = B[k * sbk + j * sbj]; C(i, j) = C[i * ldc + j] (row-major) or C[i + j * ldc]
    long long   off_stride, col_stride, val_stride, b_stride, c_stride;   // between the matrices of a batch (0 = shared)
    int         brows, bnnz, bs, n, base, ch, nchunks;
    int         a_row, c_row, c_f32;    // blocks row-major, C row-major, 16-bit A / B into an fp32 C
    int         ntiles;                 // column tiles of C per block-row tile
};

// the first piece boundary at or after stored block x: a block-row start, or a block-row start plus a multiple of ch
__device__ __forceinline__ int mm_cut_ge(const SpmmBsrArgs& a, const int* off, int x) {
    if (x >= a.bnnz) return a.bnnz;
    const int r = csr_row_of(off, a.brows, a.base, x);
    const int rs = __ldg(off + r) - a.base, re = __ldg(off + r + 1) - a.base;
    const long long c = rs + (long long)((x - rs + a.ch - 1) / a.ch) * a.ch;
    return (int)(c < re ? c : re);
}

// The walk over stored blocks: the block-row being walked and the start of the current piece.
struct MmWalk {
    int r, rs, re, ps;
    __device__ __forceinline__ void at(const SpmmBsrArgs& a, const int* off, int e) {
        r = csr_row_of(off, a.brows, a.base, e);
        rs = __ldg(off + r) - a.base; re = __ldg(off + r + 1) - a.base; ps = e;
    }
    // does stored block e end a piece?
    __device__ __forceinline__ bool cut(const SpmmBsrArgs& a, int e) const { return e + 1 == re || (e + 1 - rs) % a.ch == 0; }
    __device__ __forceinline__ bool direct(const SpmmBsrArgs& a) const { return a.carry == nullptr || re - rs <= a.ch; }
    // carry slot of the current piece: 2 per chunk, [0] a piece of a row begun in an earlier chunk, [1] the first piece of a long row
    __device__ __forceinline__ long long slot(const SpmmBsrArgs& a, long long bi) const {
        return bi * 2 * a.nchunks + 2 * (ps / a.ch) + (ps == rs ? 1 : 0);
    }
    __device__ __forceinline__ void next(const SpmmBsrArgs& a, const int* off, int e) {
        ps = e + 1;
        if (e + 1 == re)
            while (r + 1 < a.brows) {                                 // the next block-row that stores something
                r++; rs = re; re = __ldg(off + r + 1) - a.base;
                if (re > rs) break;
            }
    }
};

// The CTA's stored blocks [S, E): the pieces starting in chunk blockIdx.x (split walk) or block-row blockIdx.x (unsplit walk).
// false: nothing to multiply (a chunk inside one piece, or an empty block-row, whose beta * C the caller writes in the unsplit walk).
__device__ __forceinline__ bool mm_range(const SpmmBsrArgs& a, const int* off, int& S, int& E) {
    const int u = (int)blockIdx.x;
    if (a.carry) {
        S = mm_cut_ge(a, off, u * a.ch);
        const long long x = (long long)(u + 1) * a.ch;
        E = mm_cut_ge(a, off, x < a.bnnz ? (int)x : a.bnnz);
    } else {
        S = a.bnnz == 0 ? 0 : __ldg(off + u) - a.base;
        E = a.bnnz == 0 ? 0 : __ldg(off + u + 1) - a.base;
    }
    return S < E;
}

// C entry (row i of the matrix, column j) = alpha * acc + beta * C, rounded once to C's type (T, or fp32 when c_f32)
template <typename T, typename S>
__device__ __forceinline__ void mm_store(const SpmmBsrArgs& a, long long bi, long long i, long long j, S acc, S alpha, S beta) {
    const long long o = bi * a.c_stride + (a.c_row ? i * a.ldc + j : i + j * a.ldc);
    if (std::is_same<T, double>::value || std::is_same<T, float>::value || a.c_f32) {
        using TC = typename std::conditional<std::is_same<T, double>::value, double, float>::type;
        TC* p = (TC*)a.C + o;
        *p = beta == S(0) ? alpha * acc : alpha * acc + beta * *p;
    } else {
        T* p = (T*)a.C + o;
        const float v = beta == S(0) ? alpha * acc : alpha * acc + beta * to_acc(*p);
        if constexpr (std::is_same<T, __half>::value) *p = __float2half_rn(v);
        else if constexpr (std::is_same<T, __nv_bfloat16>::value) *p = __float2bfloat16_rn(v);
    }
}

// beta * C (0 for beta == 0, C not read) on rows [i0, i1) of block-row r and columns [j0, j1), in C's storage order
template <typename T, typename S>
__device__ __forceinline__ void mm_scale(const SpmmBsrArgs& a, long long bi, int r, int i0, int i1, int j0, int j1, S alpha, S beta,
                                         int tid, int nthreads) {
    const int h = i1 - i0, w = j1 - j0;
    for (int x = tid; x < h * w; x += nthreads) {
        const int i = a.c_row ? x / w : x % h, j = a.c_row ? x % w : x / h;
        mm_store<T, S>(a, bi, (long long)r * a.bs + i0 + i, j0 + j, S(0), alpha, beta);
    }
}

// One accumulator entry at the end of a piece (row lr of the block-row, column j < n): a direct row adds the piece to tot and, at
// the row's end, writes C; a piece of a long row goes to its carry slot.
template <typename T, typename S>
__device__ __forceinline__ void mm_flush(const SpmmBsrArgs& a, const MmWalk& w, long long bi, bool direct, bool row_end, int lr, int j,
                                         S& acc, S& tot, S alpha, S beta) {
    if (direct) {
        tot += acc;
        if (row_end && j < a.n) mm_store<T, S>(a, bi, (long long)w.r * a.bs + lr, j, tot, alpha, beta);
        if (row_end) tot = S(0);
    } else if (j < a.n) {
        ((S*)a.carry)[(w.slot(a, bi) * a.bs + lr) * a.n + j] = acc;
    }
    acc = S(0);
}

// ------------------------------------------------------------------------------------------------ tensor path
// Blocks stored row-major (K-contiguous).  BK: op(B) K-contiguous (sbk == 1), else N-contiguous (sbj == 1).
template <typename T, int BM, int BN, bool BK>
__global__ void __launch_bounds__(SPMM_BSR_THREADS, 1) spmm_bsr_mma_kernel(const SpmmBsrArgs a, const Scalars<float> sc) {
    constexpr int KS = SPMM_BSR_KS, PAD = SPMM_BSR_PAD, SL = SPMM_BSR_SLABS, ST = SPMM_BSR_STAGES;
    constexpr int WARPS_M = BM == 16 ? 1 : 2, WARPS_N = 4 / WARPS_M;
    constexpr int WM = BM / WARPS_M, WN = BN / WARPS_N;
    constexpr int MT = WM / 16, NT = WN / 8;
    constexpr int KLD = KS + PAD, BLD = BN + PAD;
    constexpr int A_ELEMS = BM * KLD;
    constexpr int B_ELEMS = BK ? BN * KLD : KS * BLD;
    constexpr int STAGE = SL * (A_ELEMS + B_ELEMS);
    extern __shared__ __align__(16) unsigned char mm_smem[];
    T* const sm = (T*)mm_smem;

    const int tid = (int)threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int wm = warp / WARPS_N, wn = warp % WARPS_N;
    const long long bi = blockIdx.z;
    const int ti = (int)(blockIdx.y / a.ntiles) * BM, n0 = (int)(blockIdx.y % a.ntiles) * BN;
    const int* off = a.off + bi * a.off_stride;
    const int* col = a.col + bi * a.col_stride;
    const T* V = (const T*)a.val + bi * a.val_stride;
    const T* B = (const T*)a.B + bi * a.b_stride;
    const float alpha = sc.a(), beta = sc.b();
    int S, E;
    if (!mm_range(a, off, S, E)) {
        if (!a.carry) mm_scale<T, float>(a, bi, blockIdx.x, ti, ti + BM, n0, min(n0 + BN, a.n), alpha, beta, tid, SPMM_BSR_THREADS);
        return;
    }
    const int spb = a.bs / KS;                                          // slabs per block
    const int nslab = (E - S) * spb, nstage = (nslab + SL - 1) / SL;

    auto load_stage = [&](int buf, int s) {
        T* sA = sm + buf * STAGE;
        T* sB = sA + SL * A_ELEMS;
#pragma unroll
        for (int u = 0; u < SL; u++) {
            const int j = s * SL + u;
            if (j >= nslab) break;
            const long long e = S + j / spb;
            const int kofs = (j % spb) * KS;
            const T* blk = V + e * a.bs * a.bs;
            for (int x = tid; x < BM * 2; x += SPMM_BSR_THREADS) {     // BM rows x 2 chunks of 8 along K
                const int rr = x >> 1, h = x & 1;
                cp_async16(sA + u * A_ELEMS + rr * KLD + h * 8, blk + (long long)(ti + rr) * a.bs + kofs + h * 8, 16);
            }
            const long long kb = (long long)(__ldg(col + e) - a.base) * a.bs + kofs;   // first row of op(B) of the slab
            if (BK) {                                                   // BN columns x 2 chunks of 8 along K
                for (int x = tid; x < BN * 2; x += SPMM_BSR_THREADS) {
                    const int c = x >> 1, h = x & 1, jj = n0 + c;
                    const bool in = jj < a.n;
                    cp_async16(sB + u * B_ELEMS + c * KLD + h * 8, in ? B + (long long)jj * a.sbj + kb + h * 8 : B, in ? 16 : 0);
                }
            } else {                                                    // 16 rows of K x BN / 8 chunks along N, the n edge zero-filled
                for (int x = tid; x < KS * (BN / 8); x += SPMM_BSR_THREADS) {
                    const int kr = x / (BN / 8), q = x % (BN / 8), jj = n0 + q * 8;
                    const int left = a.n - jj, bytes = left >= 8 ? 16 : (left > 0 ? left * 2 : 0);
                    cp_async16(sB + u * B_ELEMS + kr * BLD + q * 8, bytes ? B + (kb + kr) * a.sbk + jj : B, bytes);
                }
            }
        }
    };

    float acc[MT][NT][4], tot[MT][NT][4];
#pragma unroll
    for (int i = 0; i < MT; i++)
#pragma unroll
        for (int j = 0; j < NT; j++)
#pragma unroll
            for (int q = 0; q < 4; q++) acc[i][j][q] = tot[i][j][q] = 0.f;

    MmWalk w;
    w.at(a, off, S);
    const int g = lane >> 2, t4 = lane & 3;
#pragma unroll
    for (int s = 0; s < ST - 1; s++) {
        if (s < nstage) load_stage(s, s);
        cp_async_commit();
    }
    for (int it = 0; it < nstage; it++) {
        cp_async_wait<ST - 2>();
        __syncthreads();                               // stage `it` landed for every thread; stage it - 1's buffer is free
        if (it + ST - 1 < nstage) load_stage((it + ST - 1) % ST, it + ST - 1);
        cp_async_commit();
        const T* sA0 = sm + (it % ST) * STAGE;
        const T* sB0 = sA0 + SL * A_ELEMS;
#pragma unroll
        for (int u = 0; u < SL; u++) {
            const int j = it * SL + u;
            if (j >= nslab) break;
            const T* sA = sA0 + u * A_ELEMS;
            const T* sB = sB0 + u * B_ELEMS;
            unsigned af[MT][4], bf[NT][2];
#pragma unroll
            for (int i = 0; i < MT; i++) ldsm_x4(sA + (wm * WM + i * 16 + (lane & 15)) * KLD + (lane >> 4) * 8, af[i]);
#pragma unroll
            for (int p = 0; p < NT / 2; p++) {
                unsigned r[4];
                if (BK) ldsm_x4(sB + (wn * WN + p * 16 + (lane & 7) + (lane >> 4) * 8) * KLD + ((lane >> 3) & 1) * 8, r);
                else ldsm_x4_trans(sB + ((lane & 7) + ((lane >> 3) & 1) * 8) * BLD + wn * WN + p * 16 + (lane >> 4) * 8, r);
                bf[2 * p][0] = r[0]; bf[2 * p][1] = r[1]; bf[2 * p + 1][0] = r[2]; bf[2 * p + 1][1] = r[3];
            }
#pragma unroll
            for (int i = 0; i < MT; i++)
#pragma unroll
                for (int jn = 0; jn < NT; jn++) mma16816<T>(acc[i][jn], af[i], bf[jn][0], bf[jn][1]);
            if ((j + 1) % spb == 0) {                  // the slab ended stored block e: the end of a piece?
                const int e = S + j / spb;
                if (w.cut(a, e)) {
                    const bool direct = w.direct(a), row_end = e + 1 == w.re;
#pragma unroll
                    for (int i = 0; i < MT; i++)
#pragma unroll
                        for (int jn = 0; jn < NT; jn++) {
                            const int lr = ti + wm * WM + i * 16 + g, c = n0 + wn * WN + jn * 8 + 2 * t4;
                            mm_flush<T, float>(a, w, bi, direct, row_end, lr, c, acc[i][jn][0], tot[i][jn][0], alpha, beta);
                            mm_flush<T, float>(a, w, bi, direct, row_end, lr, c + 1, acc[i][jn][1], tot[i][jn][1], alpha, beta);
                            mm_flush<T, float>(a, w, bi, direct, row_end, lr + 8, c, acc[i][jn][2], tot[i][jn][2], alpha, beta);
                            mm_flush<T, float>(a, w, bi, direct, row_end, lr + 8, c + 1, acc[i][jn][3], tot[i][jn][3], alpha, beta);
                        }
                    w.next(a, off, e);
                }
            }
        }
    }
    cp_async_wait<0>();
}

// ------------------------------------------------------------------------------------------------ CUDA-core path
template <typename T, typename S>
__global__ void __launch_bounds__(SPMM_BSR_FX * SPMM_BSR_FY, 1) spmm_bsr_fma_kernel(const SpmmBsrArgs a, const Scalars<S> sc) {
    constexpr int TM = SPMM_BSR_FY * SPMM_BSR_FMR;
    const int tx = (int)threadIdx.x % SPMM_BSR_FX, ty = (int)threadIdx.x / SPMM_BSR_FX;
    const long long bi = blockIdx.z;
    const int ti = (int)(blockIdx.y / a.ntiles) * TM, n0 = (int)(blockIdx.y % a.ntiles) * SPMM_BSR_FX;
    const int* off = a.off + bi * a.off_stride;
    const int* col = a.col + bi * a.col_stride;
    const T* V = (const T*)a.val + bi * a.val_stride;
    const T* B = (const T*)a.B + bi * a.b_stride;
    const S alpha = sc.a(), beta = sc.b();
    int s0, s1;
    if (!mm_range(a, off, s0, s1)) {
        if (!a.carry)
            mm_scale<T, S>(a, bi, blockIdx.x, ti, min(ti + TM, a.bs), n0, min(n0 + SPMM_BSR_FX, a.n), alpha, beta,
                           (int)threadIdx.x, SPMM_BSR_FX * SPMM_BSR_FY);
        return;
    }
    const int j = n0 + tx;
    const bool jin = j < a.n;
    bool rin[SPMM_BSR_FMR];
    S acc[SPMM_BSR_FMR], tot[SPMM_BSR_FMR];
#pragma unroll
    for (int m = 0; m < SPMM_BSR_FMR; m++) { rin[m] = ti + ty + m * SPMM_BSR_FY < a.bs; acc[m] = tot[m] = S(0); }
    const long long ri = a.a_row ? a.bs : 1, rk = a.a_row ? 1 : a.bs;          // A block (i, k) = blk[i * ri + k * rk]
    MmWalk w;
    w.at(a, off, s0);
    for (int e = s0; e < s1; e++) {
        const T* blk = V + (long long)e * a.bs * a.bs + (long long)(ti + ty) * ri;
        const T* pb = B + (long long)(__ldg(col + e) - a.base) * a.bs * a.sbk + (long long)j * a.sbj;
        for (int k = 0; k < a.bs; k++) {
            const S b = jin ? S(to_acc(__ldg(pb + (long long)k * a.sbk))) : S(0);
#pragma unroll
            for (int m = 0; m < SPMM_BSR_FMR; m++) {
                const S x = rin[m] ? S(to_acc(__ldg(blk + (long long)m * SPMM_BSR_FY * ri + k * rk))) : S(0);
                acc[m] = fma(x, b, acc[m]);
            }
        }
        if (w.cut(a, e)) {
            const bool direct = w.direct(a), row_end = e + 1 == w.re;
#pragma unroll
            for (int m = 0; m < SPMM_BSR_FMR; m++) {
                if (rin[m]) mm_flush<T, S>(a, w, bi, direct, row_end, ti + ty + m * SPMM_BSR_FY, j, acc[m], tot[m], alpha, beta);
            }
            w.next(a, off, e);
        }
    }
}

// ------------------------------------------------------------------------------------------------ split walk, part 2
// Block-rows cut into several pieces: the sum of their carry slots in ascending piece order, written once.  Block-rows that store
// nothing: beta * C.  Every other block-row was written by its one piece.
template <typename T, typename S>
__global__ void __launch_bounds__(256) spmm_bsr_fixup_kernel(const SpmmBsrArgs a, const Scalars<S> sc, int ntiles) {
    const long long bi = blockIdx.z;
    const int r = (int)blockIdx.x;
    const int* off = a.off + bi * a.off_stride;
    const int rs = a.bnnz == 0 ? 0 : __ldg(off + r) - a.base, re = a.bnnz == 0 ? 0 : __ldg(off + r + 1) - a.base;
    const int cnt = re - rs;
    if (cnt > 0 && cnt <= a.ch) return;
    const int ti = (int)(blockIdx.y / ntiles) * SPMM_BSR_FIX_M, n0 = (int)(blockIdx.y % ntiles) * SPMM_BSR_FIX_N;
    const int h = min(SPMM_BSR_FIX_M, a.bs - ti), wd = min(SPMM_BSR_FIX_N, a.n - n0);
    const S alpha = sc.a(), beta = sc.b();
    if (cnt == 0) {
        mm_scale<T, S>(a, bi, r, ti, ti + h, n0, n0 + wd, alpha, beta, (int)threadIdx.x, 256);
        return;
    }
    const S* carry = (const S*)a.carry;
    const int pieces = (cnt + a.ch - 1) / a.ch;
    for (int x = (int)threadIdx.x; x < h * wd; x += 256) {
        const int i = a.c_row ? x / wd : x % h, jj = a.c_row ? x % wd : x / h;
        const int lr = ti + i, c = n0 + jj;
        S s = S(0);
        for (int p = 0; p < pieces; p++) {
            const long long ps = rs + (long long)p * a.ch;
            const long long q = bi * 2 * a.nchunks + 2 * (ps / a.ch) + (p == 0 ? 1 : 0);
            s += carry[(q * a.bs + lr) * a.n + c];
        }
        mm_store<T, S>(a, bi, (long long)r * a.bs + lr, c, s, alpha, beta);
    }
}

// ------------------------------------------------------------------------------------------------ host side
static int mm_chunk(int64_t brows, int64_t bnnz, int64_t bs, int64_t n, int batch) {
    const int64_t avg2 = brows > 0 ? (SPMM_BSR_CHUNK_FACTOR * bnnz + brows - 1) / brows : 0;
    const double work = (double)bnnz * batch * (double)((bs + 63) / 64) * (double)((n + 127) / 128);
    const int64_t spread = (int64_t)std::min(std::ceil(work / SPMM_BSR_TARGET_CTAS), 1e15);
    return (int)std::min<int64_t>(std::max<int64_t>(SPMM_BSR_CHUNK_MIN, std::min(avg2, spread)), INT32_MAX / 2);
}
static int64_t mm_nchunks(int64_t bnnz, int ch) { return (bnnz + ch - 1) / ch; }

// bytes of carry slots of the split walk; SIZE_MAX when it does not fit
static size_t mm_workspace(int ab_type, int64_t m, int64_t n, int64_t bs, int64_t bnnz, int batch) {
    if (bs < 1 || m < bs || bnnz <= 0 || n <= 0) return 0;
    const int ch = mm_chunk(m / bs, bnnz, bs, n, batch);
    const double est = 2.0 * (double)mm_nchunks(bnnz, ch) * (double)bs * (double)n * (ab_type == MM_F64 ? 8.0 : 4.0) * batch;
    if (est > 9.0e18) return SIZE_MAX;
    return (size_t)est;
}

template <typename T, int BM, int BN, bool BK>
static void launch_mm_mma(cudaStream_t st, const dim3& grid, const SpmmBsrArgs& a, const Scalars<float>& sc) {
    constexpr int A_ELEMS = BM * (SPMM_BSR_KS + SPMM_BSR_PAD);
    constexpr int B_ELEMS = BK ? BN * (SPMM_BSR_KS + SPMM_BSR_PAD) : SPMM_BSR_KS * (BN + SPMM_BSR_PAD);
    constexpr int SMEM = SPMM_BSR_STAGES * SPMM_BSR_SLABS * (A_ELEMS + B_ELEMS) * (int)sizeof(T);
    // set once, before any capture: the attribute call is not a stream operation
    static const cudaError_t attr = cudaFuncSetAttribute(spmm_bsr_mma_kernel<T, BM, BN, BK>,
                                                         cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM);
    (void)attr;
    spmm_bsr_mma_kernel<T, BM, BN, BK><<<grid, SPMM_BSR_THREADS, SMEM, st>>>(a, sc);
}

template <typename T, int BM, int BN>
static void launch_mm_mma_bm_bn(cudaStream_t st, const dim3& grid, const SpmmBsrArgs& a, const Scalars<float>& sc, bool bk) {
    if (bk) launch_mm_mma<T, BM, BN, true>(st, grid, a, sc);
    else launch_mm_mma<T, BM, BN, false>(st, grid, a, sc);
}

template <typename T, typename S>
static int launch_mm(cudaStream_t st, SpmmBsrArgs a, const Scalars<S>& sc, bool tensor, bool bk, int batch) {
    const long long units = a.carry ? a.nchunks : a.brows;
    if (units > INT32_MAX) return -1;
    if (a.bnnz > 0) {
        if constexpr (std::is_same<S, float>::value && !std::is_same<T, float>::value) {
            if (tensor) {
                const int bm = a.bs % 64 == 0 ? 64 : a.bs % 32 == 0 ? 32 : 16, bn = a.n > 64 ? 128 : 64;
                a.ntiles = (a.n + bn - 1) / bn;
                const long long ty = (long long)(a.bs / bm) * a.ntiles;
                if (ty > 65535) return -1;
                const dim3 grid((unsigned)units, (unsigned)ty, (unsigned)batch);
                if (bm == 64) { if (bn == 128) launch_mm_mma_bm_bn<T, 64, 128>(st, grid, a, sc, bk); else launch_mm_mma_bm_bn<T, 64, 64>(st, grid, a, sc, bk); }
                else if (bm == 32) { if (bn == 128) launch_mm_mma_bm_bn<T, 32, 128>(st, grid, a, sc, bk); else launch_mm_mma_bm_bn<T, 32, 64>(st, grid, a, sc, bk); }
                else { if (bn == 128) launch_mm_mma_bm_bn<T, 16, 128>(st, grid, a, sc, bk); else launch_mm_mma_bm_bn<T, 16, 64>(st, grid, a, sc, bk); }
            }
        }
        if (!tensor) {
            constexpr int tm = SPMM_BSR_FY * SPMM_BSR_FMR;
            a.ntiles = (a.n + SPMM_BSR_FX - 1) / SPMM_BSR_FX;
            const long long ty = (long long)((a.bs + tm - 1) / tm) * a.ntiles;
            if (ty > 65535) return -1;
            spmm_bsr_fma_kernel<T, S><<<dim3((unsigned)units, (unsigned)ty, (unsigned)batch), SPMM_BSR_FX * SPMM_BSR_FY, 0, st>>>(a, sc);
        }
    }
    if (a.carry || a.bnnz == 0) {                      // split walk: long block-rows and empty block-rows
        const int nt = (a.n + SPMM_BSR_FIX_N - 1) / SPMM_BSR_FIX_N;
        const long long ty = (long long)((a.bs + SPMM_BSR_FIX_M - 1) / SPMM_BSR_FIX_M) * nt;
        if (ty > 65535) return -1;
        spmm_bsr_fixup_kernel<T, S><<<dim3((unsigned)a.brows, (unsigned)ty, (unsigned)batch), 256, 0, st>>>(a, sc, nt);
    }
    return (int)cudaGetLastError();
}

}  // namespace b200

using namespace b200;

extern "C" {

void b200spmm_bsr_params(int32_t* k_slab, int32_t* slabs_per_stage, int32_t* stages, int32_t* max_rows_per_cta, int32_t* chunk_min,
                         int32_t* chunk_factor, int32_t* target_ctas) {
    if (k_slab) *k_slab = SPMM_BSR_KS;
    if (slabs_per_stage) *slabs_per_stage = SPMM_BSR_SLABS;
    if (stages) *stages = SPMM_BSR_STAGES;
    if (max_rows_per_cta) *max_rows_per_cta = SPMM_BSR_MAX_BM;
    if (chunk_min) *chunk_min = SPMM_BSR_CHUNK_MIN;
    if (chunk_factor) *chunk_factor = SPMM_BSR_CHUNK_FACTOR;
    if (target_ctas) *target_ctas = SPMM_BSR_TARGET_CTAS;
}

int b200spmm_bsr_path(int ab_type, int64_t bs, int a_row_major, const void* values, const void* B, int64_t sbk, int64_t sbj, int batch,
                      int64_t val_stride, int64_t b_stride) {
    if ((ab_type != MM_F16 && ab_type != MM_BF16) || !a_row_major) return 0;
    if (bs % SPMM_BSR_KS != 0 || ((uintptr_t)values & 15) || ((uintptr_t)B & 15)) return 0;
    if (batch > 1 && (val_stride % 8 || b_stride % 8)) return 0;
    return (sbk == 1 && sbj % 8 == 0) || (sbj == 1 && sbk % 8 == 0) ? 1 : 0;
}

size_t b200spmm_bsr_workspace_bytes(int ab_type, int64_t m, int64_t n, int64_t bs, int64_t bnnz, int batch) {
    if (batch < 1) return 0;
    return mm_workspace(ab_type, m, n, bs, bnnz, batch);
}

int b200spmm_bsr(void* stream, int ab_type, int c_type, int64_t m, int64_t k, int64_t n, int64_t bs, int64_t bnnz, const void* offsets,
                 const void* columns, const void* values, int32_t base, int a_row_major, const void* alpha, const void* beta,
                 int scalars_on_device, const void* B, int64_t sbk, int64_t sbj, void* C, int64_t ldc, int c_row_major, int batch,
                 int64_t off_stride, int64_t col_stride, int64_t val_stride, int64_t b_stride, int64_t c_stride, void* workspace,
                 size_t workspace_bytes) {
    const bool h16 = ab_type == MM_F16 || ab_type == MM_BF16;
    if (ab_type != MM_F32 && ab_type != MM_F64 && !h16) return -1;
    if (h16 ? (c_type != ab_type && c_type != MM_F32) : c_type != ab_type) return -1;
    if (m < 0 || k < 0 || n < 0 || bs < 1 || bnnz < 0 || !alpha || !beta || (base != 0 && base != 1)) return -1;
    if (m % bs || k % bs) return -1;
    if (batch < 1 || batch > 65535) return -1;
    if (sbk < 0 || sbj < 0 || off_stride < 0 || col_stride < 0 || val_stride < 0 || b_stride < 0 || c_stride < 0) return -1;
    if (m > INT32_MAX - 64 || k > INT32_MAX - 64 || n > INT32_MAX - 64 || bnnz > INT32_MAX / 2 || bs > 65536) return -1;
    if (bnnz > (m / bs) * (k / bs)) return -1;
    if (ldc < 1 || ldc < (c_row_major ? n : m)) return -1;
    if (batch > 1 && c_stride < (c_row_major ? m : n) * ldc) return -1;   // the batch's outputs would overlap
    if (m == 0 || n == 0) return 0;
    if (!C || (bnnz > 0 && (!offsets || !columns || !values || !B))) return -1;
    if (batch == 1) off_stride = col_stride = val_stride = b_stride = c_stride = 0;
    SpmmBsrArgs a;
    a.off = (const int*)offsets; a.col = (const int*)columns; a.val = values; a.B = B; a.C = C; a.carry = nullptr;
    a.sbk = sbk; a.sbj = sbj; a.ldc = ldc;
    a.off_stride = off_stride; a.col_stride = col_stride; a.val_stride = val_stride; a.b_stride = b_stride; a.c_stride = c_stride;
    a.brows = (int)(m / bs); a.bnnz = (int)bnnz; a.bs = (int)bs; a.n = (int)n; a.base = base;
    a.ch = mm_chunk(a.brows, bnnz, bs, n, batch); a.nchunks = (int)mm_nchunks(bnnz, a.ch);
    a.a_row = a_row_major != 0; a.c_row = c_row_major != 0; a.c_f32 = h16 && c_type == MM_F32; a.ntiles = 1;
    // the split walk needs the carry slots in the caller's buffer; a NULL, misaligned or small buffer gets the unsplit walk
    const size_t need = mm_workspace(ab_type, m, n, bs, bnnz, batch);
    if (need > 0 && need != SIZE_MAX && workspace_usable(workspace, workspace_bytes, need)) a.carry = workspace;
    const cudaStream_t st = (cudaStream_t)stream;
    if (ab_type == MM_F64) {
        Scalars<double> sd;
        set_scalars(sd, alpha, beta, scalars_on_device);
        return launch_mm<double, double>(st, a, sd, false, false, batch);
    }
    Scalars<float> sc;
    set_scalars(sc, alpha, beta, scalars_on_device);
    if (ab_type == MM_F32) return launch_mm<float, float>(st, a, sc, false, false, batch);
    const bool tensor = b200spmm_bsr_path(ab_type, bs, a_row_major, values, B, sbk, sbj, batch, val_stride, b_stride) == 1;
    const bool bk = sbk == 1 && sbj % 8 == 0;
    if (ab_type == MM_F16) return launch_mm<__half, float>(st, a, sc, tensor, bk, batch);
    return launch_mm<__nv_bfloat16, float>(st, a, sc, tensor, bk, batch);
}

}  // extern "C"
