// spmm_bell.cu -- Blocked-ELL x dense  C = alpha * A * B + beta * C  on H100 (sm_90a), A and B fp16 or bf16, C the same 16-bit
// type or fp32, fp32 accumulation, int32 block-column indices.  Replaces the closed library behind cusparseSpMM for Blocked-ELL
// descriptors (cuSPARSE/spmm_blockedell/spmm_blockedell_example.cpp).
//
// Format: A is rows x cols in blocks of bs x bs.  colInd holds (rows / bs) x (ellCols / bs) block columns, row-major, -1 for an
// empty slot anywhere in a block-row; values holds rows x ellCols, row-major, row r storing its block-row's blocks side by side.
// Element (r, q) of slot j is values[r * ellCols + j * bs + q] and multiplies row colInd[r / bs][j] * bs + q of B.  An empty
// slot's values are never read, and neither are B rows no block references.
//
//   * Tensor path (bs % 16 == 0, values / B 16-byte aligned, ldb % 8 == 0): bell_mma_kernel.  A CTA of 4 warps owns BM rows of
//     one block-row (BM = 64, 32 or 16, whichever divides bs) and BELL_BN columns of C.  It walks the block-row's slots in order,
//     skipping -1 without a load, and stages each 16-wide K slab of a stored block -- the BM x 16 piece of A and the 16 x BN
//     slice of B -- into shared memory with cp.async, BELL_STAGES slabs in flight.  ldmatrix (ldmatrix.trans for a row-major B)
//     feeds mma.sync.m16n8k16 with fp32 accumulators.  N-tiles are the fast grid index, so the CTAs sharing one A panel run
//     together and read it from L2.  A slab reuses a B slice only BM times: about bs flop per byte of B gathered, far below the
//     HBM ridge, so wgmma / TMA would not raise the bound.
//   * Scalar path (every other bs, and operands the 16-byte cp.async cannot take): bell_scalar_kernel, one thread per entry of
//     C, fp32 fma over the row's stored blocks in order.  The fast thread index runs along C's contiguous dimension.
// Both write each C entry once with alpha / beta applied in fp32 (beta == 0 never reads C), in a fixed order: no atomics, and
// repeated calls give identical bits.  A column-major C leaves the tensor path through a shared-memory tile in column segments.
#include <cuda_bf16.h>
#include <cuda_fp16.h>

#include <type_traits>

#include "mma_sm90.cuh"
#include "spmv_common.cuh"
#include "../../include/b200spmv.h"

namespace b200 {

constexpr int BELL_BN = 64;          // columns of C per CTA (tensor path)
constexpr int BELL_STAGES = 4;       // K slabs in flight
constexpr int BELL_KS = 16;          // K of one slab = K of one mma
constexpr int BELL_THREADS = 128;
constexpr int BELL_MAX_BM = 64;      // rows of C per CTA at most (tensor path)
constexpr int BELL_A_LD = 24;        // shared-memory row pitch (halves) of a K-contiguous slab: ldmatrix without bank conflicts
constexpr int BELL_B_LD = BELL_BN + 8;   // the same for a row-major B slice
constexpr int BELL_SC_X = 32, BELL_SC_Y = 8;   // scalar path: threads along C's contiguous dimension / along the other

constexpr int DT_F32 = 0, DT_F16 = 2, DT_BF16 = 14;   // cudaDataType values

struct BellArgs {
    const int* colind;
    const void* val;
    const void* B;
    void*       C;
    long long   ell_cols, ldb, ldc;
    int         rows, n, bs, eb, base;      // eb: slots per block-row
    int         c_f32, b_row, c_row;
    Scalars<float> s;
};

__device__ __forceinline__ float to_f(__half v) { return __half2float(v); }
__device__ __forceinline__ float to_f(__nv_bfloat16 v) { return __bfloat162float(v); }

// C(i, j) = alpha * acc + beta * C(i, j), rounded once to C's type
template <typename T>
__device__ __forceinline__ void bell_store(const BellArgs& a, long long i, long long j, float acc, float alpha, float beta) {
    const long long o = a.c_row ? i * a.ldc + j : i + j * a.ldc;
    if (a.c_f32) {
        float* p = (float*)a.C + o;
        *p = beta == 0.f ? alpha * acc : alpha * acc + beta * *p;
    } else {
        T* p = (T*)a.C + o;
        const float v = beta == 0.f ? alpha * acc : alpha * acc + beta * to_f(*p);
        if constexpr (std::is_same<T, __half>::value) *p = __float2half_rn(v);
        else *p = __float2bfloat16_rn(v);
    }
}

// ------------------------------------------------------------------------------------------------ scalar path
template <typename T, bool ROWS_FAST>
__global__ void __launch_bounds__(BELL_SC_X * BELL_SC_Y) bell_scalar_kernel(const BellArgs a) {
    const long long tiles_fast = ROWS_FAST ? (a.rows + BELL_SC_X - 1) / BELL_SC_X : (a.n + BELL_SC_X - 1) / BELL_SC_X;
    const long long t = blockIdx.x;
    const long long f = (t % tiles_fast) * BELL_SC_X + threadIdx.x, s = (t / tiles_fast) * BELL_SC_Y + threadIdx.y;
    const long long i = ROWS_FAST ? f : s, j = ROWS_FAST ? s : f;
    if (i >= a.rows || j >= a.n) return;
    const T* B = (const T*)a.B;
    const int* ci = a.colind + (i / a.bs) * a.eb;
    const T* av = (const T*)a.val + i * a.ell_cols;
    const long long sk = a.b_row ? a.ldb : 1;                       // B(k, j) = B[k * sk + j * sj]
    const long long sj = a.b_row ? 1 : a.ldb;
    float acc = 0.f;
    for (int e = 0; e < a.eb; e++) {
        const int c = __ldg(ci + e);
        if (c == -1) continue;
        const T* ap = av + (long long)e * a.bs;
        const T* bp = B + (long long)(c - a.base) * a.bs * sk + j * sj;
        for (int q = 0; q < a.bs; q++) acc = fmaf(to_f(ap[q]), to_f(bp[q * sk]), acc);
    }
    bell_store<T>(a, i, j, acc, a.s.a(), a.s.b());
}

// ------------------------------------------------------------------------------------------------ tensor path
template <typename T, int BM, bool BROW>
__global__ void __launch_bounds__(BELL_THREADS) bell_mma_kernel(const BellArgs a) {
    constexpr int WARPS_M = BM == 16 ? 1 : 2, WARPS_N = 4 / WARPS_M;
    constexpr int WM = BM / WARPS_M, WN = BELL_BN / WARPS_N;
    constexpr int MT = WM / 16, NT = WN / 8;
    constexpr int A_ELEMS = BM * BELL_A_LD;
    constexpr int B_ELEMS = BROW ? BELL_KS * BELL_B_LD : BELL_BN * BELL_A_LD;
    __shared__ __align__(16) T sA[BELL_STAGES][A_ELEMS];
    __shared__ __align__(16) T sB[BELL_STAGES][B_ELEMS];
    __shared__ float sC[BM][BELL_BN + 1];

    const int tid = (int)threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int wm = warp / WARPS_N, wn = warp % WARPS_N;
    const int tiles_n = (a.n + BELL_BN - 1) / BELL_BN;
    const long long row0 = (long long)(blockIdx.x / tiles_n) * BM;
    const int n0 = (int)(blockIdx.x % tiles_n) * BELL_BN;
    const int* ci = a.colind + (row0 / a.bs) * a.eb;
    const T* Av = (const T*)a.val;
    const T* B = (const T*)a.B;

    // stored blocks of this block-row -> K slabs in the pipeline
    int live = 0;
    for (int e0 = 0; e0 < a.eb; e0 += BELL_THREADS) {
        const int e = e0 + tid;
        live += __syncthreads_count(e < a.eb && __ldg(ci + e) != -1);
    }
    const int per_block = a.bs / BELL_KS;
    const int nslab = live * per_block;

    // the producer walks (slot, k offset) over stored blocks only, in slot order; every thread walks it the same way
    int pe = 0, pk = 0;
    while (pe < a.eb && __ldg(ci + pe) == -1) pe++;
    auto load_slab = [&](int buf) {
        const long long kb = (long long)(__ldg(ci + pe) - a.base) * a.bs + pk;     // first B row of the slab
        for (int x = tid; x < BM * 2; x += BELL_THREADS) {                         // A: BM rows x 2 chunks of 8
            const int r = x >> 1, u = x & 1;
            cp_async16(&sA[buf][r * BELL_A_LD + u * 8], Av + (row0 + r) * a.ell_cols + (long long)pe * a.bs + pk + u * 8, 16);
        }
        if (BROW) {                                                                // B: 16 rows x 8 chunks, row pitch BELL_B_LD
            const int r = tid >> 3, u = tid & 7, j = n0 + u * 8;
            const int left = a.n - j, bytes = left >= 8 ? 16 : (left > 0 ? left * 2 : 0);
            cp_async16(&sB[buf][r * BELL_B_LD + u * 8], bytes ? B + (kb + r) * a.ldb + j : B, bytes);
        } else {                                                                   // B: BN columns x 2 chunks (K-contiguous)
            for (int x = tid; x < BELL_BN * 2; x += BELL_THREADS) {
                const int c = x >> 1, u = x & 1, j = n0 + c;
                cp_async16(&sB[buf][c * BELL_A_LD + u * 8], j < a.n ? B + (long long)j * a.ldb + kb + u * 8 : B, j < a.n ? 16 : 0);
            }
        }
        pk += BELL_KS;
        if (pk == a.bs) {
            pk = 0;
            do pe++; while (pe < a.eb && __ldg(ci + pe) == -1);
        }
    };

    float acc[MT][NT][4];
#pragma unroll
    for (int i = 0; i < MT; i++)
#pragma unroll
        for (int j = 0; j < NT; j++)
#pragma unroll
            for (int q = 0; q < 4; q++) acc[i][j][q] = 0.f;

#pragma unroll
    for (int s = 0; s < BELL_STAGES - 1; s++) {
        if (s < nslab) load_slab(s);
        cp_async_commit();
    }
    for (int it = 0; it < nslab; it++) {
        cp_async_wait<BELL_STAGES - 2>();
        __syncthreads();                               // slab `it` landed for every thread; slab it - 1's buffer is free
        if (it + BELL_STAGES - 1 < nslab) load_slab((it + BELL_STAGES - 1) % BELL_STAGES);
        cp_async_commit();
        const int buf = it % BELL_STAGES;
        unsigned af[MT][4], bf[NT][2];
#pragma unroll
        for (int i = 0; i < MT; i++)
            ldsm_x4(&sA[buf][(wm * WM + i * 16 + (lane & 15)) * BELL_A_LD + (lane >> 4) * 8], af[i]);
#pragma unroll
        for (int p = 0; p < NT / 2; p++) {
            unsigned r[4];
            if (BROW) ldsm_x4_trans(&sB[buf][((lane & 7) + ((lane >> 3) & 1) * 8) * BELL_B_LD + wn * WN + p * 16 + (lane >> 4) * 8], r);
            else ldsm_x4(&sB[buf][(wn * WN + p * 16 + (lane & 7) + (lane >> 4) * 8) * BELL_A_LD + ((lane >> 3) & 1) * 8], r);
            bf[2 * p][0] = r[0]; bf[2 * p][1] = r[1]; bf[2 * p + 1][0] = r[2]; bf[2 * p + 1][1] = r[3];
        }
#pragma unroll
        for (int i = 0; i < MT; i++)
#pragma unroll
            for (int j = 0; j < NT; j++) mma16816<T>(acc[i][j], af[i], bf[j][0], bf[j][1]);
    }
    cp_async_wait<0>();

    // epilogue: the CTA's BM x BN tile through shared memory, then out along C's contiguous dimension
    const int g = lane >> 2, t4 = lane & 3;
#pragma unroll
    for (int i = 0; i < MT; i++)
#pragma unroll
        for (int j = 0; j < NT; j++) {
            const int r = wm * WM + i * 16 + g, c = wn * WN + j * 8 + 2 * t4;
            sC[r][c] = acc[i][j][0]; sC[r][c + 1] = acc[i][j][1];
            sC[r + 8][c] = acc[i][j][2]; sC[r + 8][c + 1] = acc[i][j][3];
        }
    __syncthreads();
    const float alpha = a.s.a(), beta = a.s.b();
    for (int x = tid; x < BM * BELL_BN; x += BELL_THREADS) {
        const int r = a.c_row ? x / BELL_BN : x % BM, c = a.c_row ? x % BELL_BN : x / BM;
        if (n0 + c < a.n) bell_store<T>(a, row0 + r, n0 + c, sC[r][c], alpha, beta);
    }
}

template <typename T>
static int launch_bell(cudaStream_t st, const BellArgs& a, bool tensor) {
    if (tensor) {
        const long long tiles_n = (a.n + BELL_BN - 1) / BELL_BN;
        const int bm = a.bs % 64 == 0 ? 64 : a.bs % 32 == 0 ? 32 : 16;
        const long long grid = (long long)(a.rows / bm) * tiles_n;
        if (grid > INT32_MAX) return -1;
#define B200_BELL_MMA(BM)                                                                                     \
    if (a.b_row) bell_mma_kernel<T, BM, true><<<(unsigned)grid, BELL_THREADS, 0, st>>>(a);                 \
    else bell_mma_kernel<T, BM, false><<<(unsigned)grid, BELL_THREADS, 0, st>>>(a);
        if (bm == 64) { B200_BELL_MMA(64) } else if (bm == 32) { B200_BELL_MMA(32) } else { B200_BELL_MMA(16) }
#undef B200_BELL_MMA
        return (int)cudaGetLastError();
    }
    const bool rows_fast = !a.c_row;                    // column-major C: a warp writes 32 consecutive rows of one column
    const long long fast = rows_fast ? a.rows : a.n, slow = rows_fast ? a.n : a.rows;
    const long long grid = ((fast + BELL_SC_X - 1) / BELL_SC_X) * ((slow + BELL_SC_Y - 1) / BELL_SC_Y);
    if (grid > INT32_MAX) return -1;
    const dim3 blk(BELL_SC_X, BELL_SC_Y);
    if (rows_fast) bell_scalar_kernel<T, true><<<(unsigned)grid, blk, 0, st>>>(a);
    else bell_scalar_kernel<T, false><<<(unsigned)grid, blk, 0, st>>>(a);
    return (int)cudaGetLastError();
}

}  // namespace b200

using namespace b200;

extern "C" {

void b200spmm_bell_params(int32_t* n_tile, int32_t* stages, int32_t* max_rows_per_cta) {
    if (n_tile) *n_tile = BELL_BN;
    if (stages) *stages = BELL_STAGES;
    if (max_rows_per_cta) *max_rows_per_cta = BELL_MAX_BM;
}

int b200spmm_bell(void* stream, int a_type, int c_type, int64_t rows, int64_t cols, int64_t n, int64_t bs, int64_t ell_cols,
                  const void* col_ind, const void* values, int32_t base, const void* alpha, const void* beta, int scalars_on_device,
                  const void* B, int64_t ldb, int b_row_major, void* C, int64_t ldc, int c_row_major) {
    if (a_type != DT_F16 && a_type != DT_BF16) return -1;
    if (c_type != a_type && c_type != DT_F32) return -1;
    if (rows < 0 || cols < 0 || n < 0 || bs < 1 || ell_cols < 0 || !alpha || !beta || (base != 0 && base != 1)) return -1;
    if (rows % bs || cols % bs || ell_cols % bs || ell_cols > cols) return -1;
    if (rows > INT32_MAX || cols > INT32_MAX || n > INT32_MAX || bs > INT32_MAX / 2) return -1;
    if (ldb < (b_row_major ? n : cols) || ldc < (c_row_major ? n : rows) || ldb < 1 || ldc < 1) return -1;
    if (rows == 0 || n == 0) return 0;
    if (!C || (ell_cols > 0 && (!col_ind || !values || !B))) return -1;
    BellArgs a;
    a.colind = (const int*)col_ind; a.val = values; a.B = B; a.C = C;
    a.ell_cols = ell_cols; a.ldb = ldb; a.ldc = ldc;
    a.rows = (int)rows; a.n = (int)n; a.bs = (int)bs; a.eb = (int)(ell_cols / bs); a.base = base;
    a.c_f32 = c_type == DT_F32; a.b_row = b_row_major != 0; a.c_row = c_row_major != 0;
    if (scalars_on_device) { a.s.alpha = 0.f; a.s.beta = 0.f; a.s.alpha_dev = (const float*)alpha; a.s.beta_dev = (const float*)beta; }
    else { a.s.alpha = *(const float*)alpha; a.s.beta = *(const float*)beta; a.s.alpha_dev = nullptr; a.s.beta_dev = nullptr; }
    // the 16-byte cp.async of the tensor path needs aligned panels of A and B; every other operand takes the scalar path
    const bool tensor = bs % BELL_KS == 0 && ((uintptr_t)values & 15) == 0 && ((uintptr_t)B & 15) == 0 && ldb % 8 == 0;
    if (a_type == DT_F16) return launch_bell<__half>((cudaStream_t)stream, a, tensor);
    return launch_bell<__nv_bfloat16>((cudaStream_t)stream, a, tensor);
}

}  // extern "C"
