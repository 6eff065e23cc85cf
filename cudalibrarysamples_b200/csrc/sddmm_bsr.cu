// sddmm_bsr.cu -- sampled dense-dense product  C = alpha * (op(A) * op(B)) o spy(C) + beta * C  on H100 (sm_90a) for a BSR C:
// int32 block offsets / block columns, square bs x bs blocks stored row- or column-major inside each block, A and B dense.
// Replaces the closed library behind cusparseSDDMM for BSR descriptors (cuSPARSE/sddmm_bsr/sddmm_bsr_example.c).
//
// Every dense layout is reduced to element strides as for CSR (sddmm_csr.cu): op(A)(i, k) = A[i * sai + k * sak] and
// op(B)(k, j) = B[k * sbk + j * sbj].  Stored block e of block-row r and block column c is the small dense product
// op(A)[r*bs .. r*bs+bs, :] . op(B)[:, c*bs .. c*bs+bs]: the Q . K^T of block-sparse attention.
//
//   * Tensor path (fp16 / bf16 A and B, C of that type or fp32, bs % 16 == 0, 16-byte aligned operands, each operand contiguous
//     along K or along its other dimension with the other stride a multiple of 8): sddmm_bsr_mma_kernel.  A CTA owns one TILE x TILE
//     tile of one stored block (TILE = 64, 32 or 16, the largest that divides bs; a bs = 128 block is four CTAs split along its rows
//     and columns, never along K).  Its block-row comes from one binary search over the block offsets.  16-wide K slabs of the
//     tile's op(A) rows and op(B) columns stream through a BSR_STAGES-deep cp.async pipeline; the K edge is zero-filled through the
//     cp.async source size, so nothing past K is read.  ldmatrix (.trans for an operand that is not K-contiguous, e.g. the sample's
//     K x N row-major B) feeds mma.sync.m16n8k16 with fp32 accumulators.  Each op(B) slab is reused TILE times: about bs flop per
//     byte gathered, so the product is bound by that gather and wgmma / TMA would not raise the bound.
//   * CUDA-core path (fp32 with FFMA, fp64 with DFMA, no TF32; every bs; 16-bit operands the tensor path cannot take):
//     sddmm_bsr_fma_kernel.  A thread owns an MR x MR piece of a block (MR = 4, 2 or 1, whichever divides bs) and walks K once,
//     reusing each loaded value of op(A) / op(B) MR times; a tile is at most 16 MR x 16 MR, and a CTA holds as many whole tiles as
//     fit 256 threads (128 blocks of bs = 2, 16 of bs = 8, one 64 x 64 tile).
// Both paths read only the rows of op(A) a stored block-row references and the columns of op(B) a stored block references, write
// each C entry exactly once in a fixed k order (no atomics: repeated calls and graph replays give identical bits), round it once to
// C's type, and never read C when beta == 0.  A strided batch is one launch (blockIdx.y).  No workspace, no allocation, no host sync.
#include "mma_sm90.cuh"
#include "spmv_common.cuh"
#include "../../include/b200spmv.h"

namespace b200 {

constexpr int BSR_KS = 16;            // K of one slab = K of one mma (tensor path)
constexpr int BSR_STAGES = 4;         // K slabs in flight (tensor path)
constexpr int BSR_MAX_TILE = 64;      // widest block one CTA owns whole; wider blocks are split into 64 x 64 tiles
constexpr int BSR_PAD = 8;            // halves of row padding in shared memory: ldmatrix rows land in distinct banks
constexpr int BSR_FMA_THREADS = 256;  // CUDA-core path: threads per CTA

constexpr int DT_F32 = 0, DT_F64 = 1, DT_F16 = 2, DT_BF16 = 14;   // cudaDataType values

struct BsrArgs {
    const int* off;
    const int* col;
    void*      val;
    const void* A;
    const void* B;
    long long  sai, sak, sbk, sbj;                                  // element strides of op(A)(i, k) and op(B)(k, j)
    long long  off_stride, col_stride, val_stride, a_stride, b_stride;   // between the matrices of a batch (0 = shared)
    int        brows, bnnz, bs, k, base, c_row, c_f32;
    int        tiles;                                               // tiles per block side
};

// C entry = alpha * acc + beta * C entry, rounded once to C's type (T, or fp32 when c_f32)
template <typename T, typename S>
__device__ __forceinline__ void bsr_store(void* V, long long o, bool c_f32, S acc, S alpha, S beta) {
    if (std::is_same<T, double>::value || std::is_same<T, float>::value || c_f32) {
        using TC = typename std::conditional<std::is_same<T, double>::value, double, float>::type;
        TC* p = (TC*)V + o;
        *p = beta == S(0) ? alpha * acc : alpha * acc + beta * *p;
    } else {
        T* p = (T*)V + o;
        const float v = beta == S(0) ? alpha * acc : alpha * acc + beta * to_acc(*p);
        if constexpr (std::is_same<T, __half>::value) *p = __float2half_rn(v);
        else if constexpr (std::is_same<T, __nv_bfloat16>::value) *p = __float2bfloat16_rn(v);
    }
}

// ------------------------------------------------------------------------------------------------ tensor path
// AK: op(A) is K-contiguous (sak == 1), else M-contiguous (sai == 1); BK: op(B) is K-contiguous (sbk == 1), else N-contiguous.
template <typename T, int TILE, bool AK, bool BK>
__global__ void __launch_bounds__(TILE == 16 ? 32 : 128) sddmm_bsr_mma_kernel(const BsrArgs a, const Scalars<float> sc) {
    constexpr int THREADS = TILE == 16 ? 32 : 128;
    constexpr int WARPS_N = TILE == 16 ? 1 : 2;
    constexpr int WM = TILE == 16 ? 16 : TILE / 2, WN = TILE == 16 ? 16 : TILE / 2;
    constexpr int MT = WM / 16, NT = WN / 8;
    constexpr int KLD = BSR_KS + BSR_PAD;          // row pitch of a slab stored [TILE][16] (K-contiguous)
    constexpr int TLD = TILE + BSR_PAD;            // row pitch of a slab stored [16][TILE]
    constexpr int A_ELEMS = AK ? TILE * KLD : BSR_KS * TLD;
    constexpr int B_ELEMS = BK ? TILE * KLD : BSR_KS * TLD;
    __shared__ __align__(16) T sA[BSR_STAGES][A_ELEMS];
    __shared__ __align__(16) T sB[BSR_STAGES][B_ELEMS];
    __shared__ float sC[TILE][TILE + 1];

    const int tid = (int)threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int wm = warp / WARPS_N, wn = warp % WARPS_N;
    const int tiles2 = a.tiles * a.tiles;
    const int e = (int)(blockIdx.x / tiles2), t = (int)(blockIdx.x % tiles2);
    const long long bi = blockIdx.y;
    const int br = csr_row_of(a.off + bi * a.off_stride, a.brows, a.base, e);
    const int bc = __ldg(a.col + bi * a.col_stride + e) - a.base;
    const int ti = (t / a.tiles) * TILE, tj = (t % a.tiles) * TILE;     // the tile inside the block
    const long long r0 = (long long)br * a.bs + ti, c0 = (long long)bc * a.bs + tj;
    const T* A = (const T*)a.A + bi * a.a_stride;
    const T* B = (const T*)a.B + bi * a.b_stride;
    const int nslab = (a.k + BSR_KS - 1) / BSR_KS;

    auto load_slab = [&](int buf, int s) {
        const int k0 = s * BSR_KS;
        if (AK) {                                                       // TILE rows x 2 chunks of 8 along K
            for (int x = tid; x < TILE * 2; x += THREADS) {
                const int r = x >> 1, kk = k0 + (x & 1) * 8, left = a.k - kk;
                const int bytes = left >= 8 ? 16 : (left > 0 ? left * 2 : 0);
                cp_async16(&sA[buf][r * KLD + (x & 1) * 8], bytes ? A + (r0 + r) * a.sai + kk : A, bytes);
            }
        } else {                                                        // 16 rows of K x TILE / 8 chunks along M
            for (int x = tid; x < BSR_KS * (TILE / 8); x += THREADS) {
                const int kr = x / (TILE / 8), u = x % (TILE / 8);
                const bool in = k0 + kr < a.k;
                cp_async16(&sA[buf][kr * TLD + u * 8], in ? A + (long long)(k0 + kr) * a.sak + r0 + u * 8 : A, in ? 16 : 0);
            }
        }
        if (BK) {
            for (int x = tid; x < TILE * 2; x += THREADS) {
                const int c = x >> 1, kk = k0 + (x & 1) * 8, left = a.k - kk;
                const int bytes = left >= 8 ? 16 : (left > 0 ? left * 2 : 0);
                cp_async16(&sB[buf][c * KLD + (x & 1) * 8], bytes ? B + (c0 + c) * a.sbj + kk : B, bytes);
            }
        } else {
            for (int x = tid; x < BSR_KS * (TILE / 8); x += THREADS) {
                const int kr = x / (TILE / 8), u = x % (TILE / 8);
                const bool in = k0 + kr < a.k;
                cp_async16(&sB[buf][kr * TLD + u * 8], in ? B + (long long)(k0 + kr) * a.sbk + c0 + u * 8 : B, in ? 16 : 0);
            }
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
    for (int s = 0; s < BSR_STAGES - 1; s++) {
        if (s < nslab) load_slab(s, s);
        cp_async_commit();
    }
    for (int it = 0; it < nslab; it++) {
        cp_async_wait<BSR_STAGES - 2>();
        __syncthreads();                               // slab `it` landed for every thread; slab it - 1's buffer is free
        if (it + BSR_STAGES - 1 < nslab) load_slab((it + BSR_STAGES - 1) % BSR_STAGES, it + BSR_STAGES - 1);
        cp_async_commit();
        const int buf = it % BSR_STAGES;
        unsigned af[MT][4], bf[NT][2];
#pragma unroll
        for (int i = 0; i < MT; i++) {
            if (AK) ldsm_x4(&sA[buf][(wm * WM + i * 16 + (lane & 15)) * KLD + (lane >> 4) * 8], af[i]);
            else ldsm_x4_trans(&sA[buf][((lane >> 4) * 8 + (lane & 7)) * TLD + wm * WM + i * 16 + ((lane >> 3) & 1) * 8], af[i]);
        }
#pragma unroll
        for (int p = 0; p < NT / 2; p++) {
            unsigned r[4];
            if (BK) ldsm_x4(&sB[buf][(wn * WN + p * 16 + (lane & 7) + (lane >> 4) * 8) * KLD + ((lane >> 3) & 1) * 8], r);
            else ldsm_x4_trans(&sB[buf][((lane & 7) + ((lane >> 3) & 1) * 8) * TLD + wn * WN + p * 16 + (lane >> 4) * 8], r);
            bf[2 * p][0] = r[0]; bf[2 * p][1] = r[1]; bf[2 * p + 1][0] = r[2]; bf[2 * p + 1][1] = r[3];
        }
#pragma unroll
        for (int i = 0; i < MT; i++)
#pragma unroll
            for (int j = 0; j < NT; j++) mma16816<T>(acc[i][j], af[i], bf[j][0], bf[j][1]);
    }
    cp_async_wait<0>();

    // epilogue: the tile through shared memory, then out in C's block order (consecutive threads, consecutive addresses)
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
    const float alpha = sc.a(), beta = sc.b();
    const long long vbase = bi * a.val_stride + (long long)e * a.bs * a.bs;
    for (int x = tid; x < TILE * TILE; x += THREADS) {
        const int p = x / TILE, q = x % TILE;
        const int i = a.c_row ? p : q, j = a.c_row ? q : p;
        const long long o = a.c_row ? (long long)(ti + i) * a.bs + tj + j : (long long)(tj + j) * a.bs + ti + i;
        bsr_store<T>(a.val, vbase + o, a.c_f32, sC[i][j], alpha, beta);
    }
}

// ------------------------------------------------------------------------------------------------ CUDA-core path
template <typename T, typename S, int MR>
__global__ void __launch_bounds__(BSR_FMA_THREADS) sddmm_bsr_fma_kernel(const BsrArgs a, const Scalars<S> sc) {
    const int st = min(a.bs, 16 * MR);                      // tile side: at most 16 x 16 threads per tile, MR divides it
    const int per = st / MR, tpt = per * per;               // threads per tile side, per tile
    const int slot = (int)threadIdx.x / tpt, w = (int)threadIdx.x % tpt;
    const int tiles2 = a.tiles * a.tiles;
    const long long g = (long long)blockIdx.x * (BSR_FMA_THREADS / tpt) + slot;
    if (slot >= BSR_FMA_THREADS / tpt || g >= (long long)a.bnnz * tiles2) return;
    const int e = (int)(g / tiles2), t = (int)(g % tiles2);
    const long long bi = blockIdx.y;
    const int br = csr_row_of(a.off + bi * a.off_stride, a.brows, a.base, e);
    const int bc = __ldg(a.col + bi * a.col_stride + e) - a.base;
    const int i0 = (t / a.tiles) * st + (w / per) * MR, j0 = (t % a.tiles) * st + (w % per) * MR;   // inside the block
    const T* pa = (const T*)a.A + bi * a.a_stride + ((long long)br * a.bs + i0) * a.sai;
    const T* pb = (const T*)a.B + bi * a.b_stride + ((long long)bc * a.bs + j0) * a.sbj;
    bool ri[MR], cj[MR];
#pragma unroll
    for (int r = 0; r < MR; r++) { ri[r] = i0 + r < a.bs; cj[r] = j0 + r < a.bs; }
    S acc[MR][MR];
#pragma unroll
    for (int r = 0; r < MR; r++)
#pragma unroll
        for (int c = 0; c < MR; c++) acc[r][c] = S(0);
    for (int k = 0; k < a.k; k++) {
        S xa[MR], xb[MR];
#pragma unroll
        for (int r = 0; r < MR; r++) {
            xa[r] = ri[r] ? S(to_acc(__ldg(pa + r * a.sai + k * a.sak))) : S(0);
            xb[r] = cj[r] ? S(to_acc(__ldg(pb + r * a.sbj + k * a.sbk))) : S(0);
        }
#pragma unroll
        for (int r = 0; r < MR; r++)
#pragma unroll
            for (int c = 0; c < MR; c++) acc[r][c] = fma(xa[r], xb[c], acc[r][c]);
    }
    const S alpha = sc.a(), beta = sc.b();
    const long long vbase = bi * a.val_stride + (long long)e * a.bs * a.bs;
#pragma unroll
    for (int r = 0; r < MR; r++)
#pragma unroll
        for (int c = 0; c < MR; c++)
            if (ri[r] && cj[c]) {
                const long long o = a.c_row ? (long long)(i0 + r) * a.bs + j0 + c : (long long)(j0 + c) * a.bs + i0 + r;
                bsr_store<T>(a.val, vbase + o, a.c_f32, acc[r][c], alpha, beta);
            }
}

template <typename T>
static int launch_bsr_mma(cudaStream_t st, BsrArgs a, const Scalars<float>& sc, bool ak, bool bk, int batch) {
    const int tile = a.bs % 64 == 0 ? 64 : a.bs % 32 == 0 ? 32 : 16;
    a.tiles = a.bs / tile;
    const long long grid = (long long)a.bnnz * a.tiles * a.tiles;
    if (grid > INT32_MAX) return -1;
    const dim3 g((unsigned)grid, (unsigned)batch);
#define B200_BSR_MMA(TILE)                                                                                         \
    {                                                                                                              \
        constexpr int th = TILE == 16 ? 32 : 128;                                                                  \
        if (ak && bk) sddmm_bsr_mma_kernel<T, TILE, true, true><<<g, th, 0, st>>>(a, sc);                          \
        else if (ak) sddmm_bsr_mma_kernel<T, TILE, true, false><<<g, th, 0, st>>>(a, sc);                          \
        else if (bk) sddmm_bsr_mma_kernel<T, TILE, false, true><<<g, th, 0, st>>>(a, sc);                          \
        else sddmm_bsr_mma_kernel<T, TILE, false, false><<<g, th, 0, st>>>(a, sc);                                 \
    }
    if (tile == 64) B200_BSR_MMA(64) else if (tile == 32) B200_BSR_MMA(32) else B200_BSR_MMA(16)
#undef B200_BSR_MMA
    return (int)cudaGetLastError();
}

template <typename T, typename S>
static int launch_bsr_fma(cudaStream_t st, BsrArgs a, const Scalars<S>& sc, int batch) {
    const int mr = a.bs % 4 == 0 ? 4 : a.bs % 2 == 0 ? 2 : 1;
    const int side = a.bs < 16 * mr ? a.bs : 16 * mr;
    a.tiles = (a.bs + side - 1) / side;
    const long long tpt = (long long)(side / mr) * (side / mr);
    const long long per_cta = BSR_FMA_THREADS / tpt;
    const long long grid = ((long long)a.bnnz * a.tiles * a.tiles + per_cta - 1) / per_cta;
    if (grid > INT32_MAX) return -1;
    const dim3 g((unsigned)grid, (unsigned)batch);
    if (mr == 4) sddmm_bsr_fma_kernel<T, S, 4><<<g, BSR_FMA_THREADS, 0, st>>>(a, sc);
    else if (mr == 2) sddmm_bsr_fma_kernel<T, S, 2><<<g, BSR_FMA_THREADS, 0, st>>>(a, sc);
    else sddmm_bsr_fma_kernel<T, S, 1><<<g, BSR_FMA_THREADS, 0, st>>>(a, sc);
    return (int)cudaGetLastError();
}

}  // namespace b200

using namespace b200;

extern "C" {

void b200sddmm_bsr_params(int32_t* k_slab, int32_t* stages, int32_t* max_tile, int32_t* fma_threads) {
    if (k_slab) *k_slab = BSR_KS;
    if (stages) *stages = BSR_STAGES;
    if (max_tile) *max_tile = BSR_MAX_TILE;
    if (fma_threads) *fma_threads = BSR_FMA_THREADS;
}

int b200sddmm_bsr_path(int ab_type, int64_t bs, const void* A, int64_t sai, int64_t sak, const void* B, int64_t sbk, int64_t sbj,
                       int batch, int64_t a_stride, int64_t b_stride) {
    if (ab_type != DT_F16 && ab_type != DT_BF16) return 0;
    if (bs % BSR_KS != 0 || ((uintptr_t)A & 15) || ((uintptr_t)B & 15)) return 0;
    if (batch > 1 && (a_stride % 8 || b_stride % 8)) return 0;
    const bool a_ok = (sak == 1 && sai % 8 == 0) || (sai == 1 && sak % 8 == 0);
    const bool b_ok = (sbk == 1 && sbj % 8 == 0) || (sbj == 1 && sbk % 8 == 0);
    return a_ok && b_ok ? 1 : 0;
}

int b200sddmm_bsr(void* stream, int ab_type, int c_type, int64_t m, int64_t n, int64_t k, int64_t bs, int64_t bnnz, const void* offsets,
                  const void* columns, void* values, int32_t base, int c_row_major, const void* alpha, const void* beta,
                  int scalars_on_device, const void* A, int64_t sai, int64_t sak, const void* B, int64_t sbk, int64_t sbj, int batch,
                  int64_t off_stride, int64_t col_stride, int64_t val_stride, int64_t a_stride, int64_t b_stride) {
    const bool h16 = ab_type == DT_F16 || ab_type == DT_BF16;
    if (ab_type != DT_F32 && ab_type != DT_F64 && !h16) return -1;
    if (h16 ? (c_type != ab_type && c_type != DT_F32) : c_type != ab_type) return -1;
    if (m < 0 || n < 0 || k < 0 || bs < 1 || bnnz < 0 || !alpha || !beta || (base != 0 && base != 1)) return -1;
    if (m % bs || n % bs) return -1;
    if (batch < 1 || batch > 65535) return -1;
    if (sai < 0 || sak < 0 || sbk < 0 || sbj < 0 || off_stride < 0 || col_stride < 0 || val_stride < 0 || a_stride < 0 || b_stride < 0)
        return -1;
    if (m > INT32_MAX - 64 || n > INT32_MAX - 64 || k > INT32_MAX - 64 || bnnz > INT32_MAX || bs > 65536) return -1;
    if (bnnz > (m / bs) * (n / bs)) return -1;
    if (batch > 1 && val_stride < bnnz * bs * bs) return -1;       // the batch's outputs would overlap
    if (m == 0 || bnnz == 0) return 0;
    if (!offsets || !columns || !values || (k > 0 && (!A || !B))) return -1;
    if (batch == 1) off_stride = col_stride = val_stride = a_stride = b_stride = 0;
    BsrArgs a;
    a.off = (const int*)offsets; a.col = (const int*)columns; a.val = values; a.A = A; a.B = B;
    a.sai = sai; a.sak = sak; a.sbk = sbk; a.sbj = sbj;
    a.off_stride = off_stride; a.col_stride = col_stride; a.val_stride = val_stride; a.a_stride = a_stride; a.b_stride = b_stride;
    a.brows = (int)(m / bs); a.bnnz = (int)bnnz; a.bs = (int)bs; a.k = (int)k; a.base = base; a.c_row = c_row_major != 0;
    a.c_f32 = h16 && c_type == DT_F32; a.tiles = 1;
    const cudaStream_t st = (cudaStream_t)stream;
    if (ab_type == DT_F64) {
        Scalars<double> sd;
        set_scalars(sd, alpha, beta, scalars_on_device);
        return launch_bsr_fma<double, double>(st, a, sd, batch);
    }
    Scalars<float> sc;
    set_scalars(sc, alpha, beta, scalars_on_device);
    if (ab_type == DT_F32) return launch_bsr_fma<float, float>(st, a, sc, batch);
    if (b200sddmm_bsr_path(ab_type, bs, A, sai, sak, B, sbk, sbj, batch, a_stride, b_stride)) {
        const bool ak = sak == 1 && sai % 8 == 0, bk = sbk == 1 && sbj % 8 == 0;
        if (ab_type == DT_F16) return launch_bsr_mma<__half>(st, a, sc, ak, bk, batch);
        return launch_bsr_mma<__nv_bfloat16>(st, a, sc, ak, bk, batch);
    }
    if (ab_type == DT_F16) return launch_bsr_fma<__half, float>(st, a, sc, batch);
    return launch_bsr_fma<__nv_bfloat16, float>(st, a, sc, batch);
}

}  // extern "C"
