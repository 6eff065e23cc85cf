// spmm_csr16.cu -- CSR x dense  C = alpha * A * op(B) + beta * C  on H100 (sm_90a) in half precision: A m x k CSR with int32
// offsets / columns (base 0 or 1) and fp16 or bf16 values, op(B) k x n of A's type, C m x n of A's type or fp32, fp32 accumulation.
// Replaces the closed library behind cusparseSpMM for a 16-bit CSR A (graph aggregation, pruned-weight inference).  op(B) is reduced
// to element strides as in spmm_bsr.cu: op(B)(k, j) = B[k * sbk + j * sbj].  Kept apart from spmm_csr.cu (fp32 / fp64), whose
// kernels stay as they are.
//
// A warp owns a row (or a piece of one) and a panel of 32 * V columns of C, V = 1, 2, 4 or 8 columns per lane chosen from n.  The
// row's (column, value) pairs are loaded 32 at a time with one coalesced instruction each and broadcast with shuffles; every lane
// then gathers its V columns of the selected B rows, SPMM_CSR16_INFLIGHT(V) rows at a time, with one V-wide load (half2 up to
// 128-bit) where the view allows it (b200spmm_csr16_path), else with scalar loads.  Each entry feeds V fp32 FMAs in entry order.
// No tensor cores: every gathered 2-byte B element feeds one FMA (about 1 flop per byte), so the gathers bound the kernel and mma
// cannot raise that bound.  A K-contiguous op(B) (column-major B, or row-major B with opB = T) is first copied row-major into the
// workspace by spmm_transpose_b_kernel, as spmm_csr.cu does, so that the gathers read contiguous rows.
//
// Row pieces.  A row is cut into pieces of at most P = SPMM_CSR16_PIECE entries at fixed positions (row start + a multiple of P).
// Split walk (workspace): the row-tile CTAs (32 rows each, 4 per warp) compute every row of one piece and write it, and the first
// piece of each longer row, which goes to a carry slot; the chunk CTAs take the later pieces: for chunk c = entries [c * P, (c + 1) *
// P) at most one such piece starts there (a row that reaches into the chunk from before it), found by one binary search over the
// offsets.  Each chunk has two carry slots, one for that later piece and one for the first piece of the long row that starts in the
// chunk (at most one does), so every slot is written once.  spmm_csr16_fixup_kernel then adds a long row's slots in ascending piece
// order, starting from 0, and writes the row once: the fix-up of chunk c owns the long row that starts in chunk c.  Unsplit walk (no
// usable workspace):
// one warp adds the same pieces in the same order (0 + s0 + s1 + ...).  So both walks give identical bits, and every C entry is
// written once without atomics: repeated calls and graph replays give identical bits.
//
// Column-major C: the row-tile CTA parks its 32 rows x 32 * V columns in shared memory and writes each column's 32 rows as one
// coalesced segment (as spmm_csr_ctile_kernel does).  The epilogue alpha * acc + beta * c is fp32 and rounds once to C's type; beta
// == 0 never reads C.  Nothing is read past n, in ld padding, or in a B row no stored entry references; an Inf / NaN in row 0 of B
// reaches only rows that store column 0.  No allocation, no host synchronisation.
#include "spmv_common.cuh"
#include "../../include/b200spmv.h"

#include <cuda_bf16.h>
#include <cuda_fp16.h>

namespace b200 {

constexpr int SPMM_CSR16_WARPS = 8;          // warps per CTA
constexpr int SPMM_CSR16_TILE_ROWS = 32;     // rows of a row-tile CTA: SPMM_CSR16_TILE_ROWS / SPMM_CSR16_WARPS per warp
constexpr int SPMM_CSR16_LANE_ENTRIES = 32;  // entries of a row loaded per coalesced batch
constexpr int SPMM_CSR16_PIECE = 512;        // P: entries per row piece
constexpr int SPMM_CSR16_MAX_V = 8;          // columns per lane at most: a panel of 256 columns
constexpr int H16_F32 = 0, H16_F16 = 2, H16_BF16 = 14;   // cudaDataType values

// B rows in flight per lane
__host__ __device__ constexpr int SPMM_CSR16_INFLIGHT(int v) { return v == 8 ? 4 : 8; }

struct SpmmCsr16Args {
    const int* off;
    const int* col;
    const void* val;
    const void* B;
    void*       C;
    float*      carry;                  // split walk: 2 * nchunks slots of n fp32 partial sums; nullptr = unsplit
    long long   sbk, sbj, ldc;          // op(B)(k, j) = B[k * sbk + j * sbj]; C(i, j) = C[i * ldc + j] (row-major) or C[i + j * ldc]
    int         rows, n, nnz, base, nchunks, ntiles;
    int         c_f32;                  // C is fp32 (else A's type)
};

__device__ __forceinline__ float h2f(__half v) { return __half2float(v); }
__device__ __forceinline__ float h2f(__nv_bfloat16 v) { return __bfloat162float(v); }

// the row holding entry x < nnz: the last r with off[r] - base <= x (an empty row never holds x)
__device__ __forceinline__ int csr16_row(const SpmmCsr16Args& a, int x) {
    int lo = 0, hi = a.rows;
    while (hi - lo > 1) {
        const int mid = (lo + hi) >> 1;
        if (__ldg(a.off + mid) - a.base <= x) lo = mid; else hi = mid;
    }
    return lo;
}

// C entry (i, j) = alpha * acc + beta * C in fp32, rounded once to C's type
template <typename T>
__device__ __forceinline__ void csr16_store(const SpmmCsr16Args& a, bool c_row, long long i, long long j, float acc, float alpha,
                                            float beta) {
    const long long o = c_row ? i * a.ldc + j : i + j * a.ldc;
    if (a.c_f32) {
        float* p = (float*)a.C + o;
        *p = beta == 0.f ? __fmul_rn(alpha, acc) : __fmaf_rn(alpha, acc, __fmul_rn(beta, *p));
    } else {
        T* p = (T*)a.C + o;
        const float v = beta == 0.f ? __fmul_rn(alpha, acc) : __fmaf_rn(alpha, acc, __fmul_rn(beta, h2f(*p)));
        if constexpr (std::is_same<T, __half>::value) *p = __float2half_rn(v);
        else *p = __float2bfloat16_rn(v);
    }
}

// Row k of op(B), columns j .. j + V - 1 (those below n; the rest 0) into h.  LW == V: one V-wide load where the lane's columns are
// all below n; LW == 1: scalar loads (a misaligned view, an odd leading dimension, or a strided op(B) without the workspace copy).
template <typename T, int V, int LW>
__device__ __forceinline__ void csr16_load_b(const SpmmCsr16Args& a, const T* B, int k, int j, T (&h)[V]) {
    const T* p = B + (long long)k * a.sbk + (long long)j * a.sbj;
    if (LW == V && LW > 1 && j + V <= a.n) {
        if constexpr (V == 8) *(uint4*)h = __ldg((const uint4*)p);
        else if constexpr (V == 4) *(uint2*)h = __ldg((const uint2*)p);
        else if constexpr (V == 2) *(unsigned*)h = __ldg((const unsigned*)p);
    } else {
#pragma unroll
        for (int q = 0; q < V; q++) {
            unsigned short bits = 0;
            if (j + q < a.n) bits = __ldg((const unsigned short*)(p + (long long)q * a.sbj));
            ((unsigned short*)h)[q] = bits;
        }
    }
}

// acc += the piece [s, e) of a row times op(B) at the lane's columns j .. j + V - 1, entry by entry in ascending order.  A lane
// whose columns are all past n loads nothing.  Slots past the piece's end take neither a load nor an FMA: an Inf or NaN in row 0 of
// B must not reach rows that do not store column 0.  s, e and so every branch on them are warp-uniform.
template <typename T, int V, int LW>
__device__ __forceinline__ void csr16_piece(const SpmmCsr16Args& a, int s, int e, int lane, int j, float (&acc)[V]) {
    constexpr int U = SPMM_CSR16_INFLIGHT(V);
    const T* B = (const T*)a.B;
    const T* vals = (const T*)a.val;
    const bool jin = j < a.n;
    for (int p = s; p < e; p += SPMM_CSR16_LANE_ENTRIES) {
        const int i = p + lane;
        const int c = i < e ? ldg_stream(a.col + i) - a.base : 0;
        const float v = i < e ? h2f(vals[i]) : 0.f;
        const int cnt = min(SPMM_CSR16_LANE_ENTRIES, e - p);
        for (int t = 0; t < cnt; t += U) {
            int kk[U];
            float vv[U];
            alignas(16) T h[U][V];
#pragma unroll
            for (int u = 0; u < U; u++) {
                kk[u] = __shfl_sync(0xffffffffu, c, (t + u) & 31);
                vv[u] = __shfl_sync(0xffffffffu, v, (t + u) & 31);
            }
#pragma unroll
            for (int u = 0; u < U; u++)
                if (jin && t + u < cnt) csr16_load_b<T, V, LW>(a, B, kk[u], j, h[u]);
#pragma unroll
            for (int u = 0; u < U; u++)
                if (jin && t + u < cnt) {
#pragma unroll
                    for (int q = 0; q < V; q++) acc[q] = __fmaf_rn(vv[u], h2f(h[u][q]), acc[q]);
                }
        }
    }
}

// carry slot of the piece starting at entry ps of a long row starting at rs: two per chunk, [0] a later piece (at most one starts in
// a chunk: that of the row reaching into it), [1] the first piece (at most one long row starts in a chunk)
__device__ __forceinline__ float* csr16_slot(const SpmmCsr16Args& a, int ps, int rs) {
    return a.carry + (2LL * (ps / SPMM_CSR16_PIECE) + (ps == rs ? 1 : 0)) * a.n;
}

template <int V>
__device__ __forceinline__ void csr16_carry(const SpmmCsr16Args& a, int ps, int rs, int j, const float (&acc)[V]) {
    float* s = csr16_slot(a, ps, rs);
#pragma unroll
    for (int q = 0; q < V; q++)
        if (j + q < a.n) s[j + q] = acc[q];
}

// blockIdx.x < ntiles: a row tile of SPMM_CSR16_TILE_ROWS rows; above (split walk only): SPMM_CSR16_WARPS chunks, one per warp.
// blockIdx.y: the panel of 32 * V columns.  CROW: C row-major (else staged through shared memory).
template <typename T, int V, int LW, bool CROW>
__global__ void __launch_bounds__(32 * SPMM_CSR16_WARPS) spmm_csr16_kernel(const SpmmCsr16Args a, const Scalars<float> sc) {
    constexpr int P = SPMM_CSR16_PIECE, PW = 32 * V, PER_WARP = SPMM_CSR16_TILE_ROWS / SPMM_CSR16_WARPS;
    const int lane = (int)threadIdx.x & 31, warp = (int)threadIdx.x >> 5;
    const int j0 = (int)blockIdx.y * PW, j = j0 + lane * V;
    float acc[V];
    if ((int)blockIdx.x >= a.ntiles) {                 // the piece p >= 1 of a long row that starts in chunk c, if there is one
        const int c = ((int)blockIdx.x - a.ntiles) * SPMM_CSR16_WARPS + warp;
        if (c >= a.nchunks) return;
        const int x = c * P;
        const int r = csr16_row(a, x);
        const int rs = __ldg(a.off + r) - a.base, re = __ldg(a.off + r + 1) - a.base;
        if (re - rs <= P) return;
        const int ps = rs + ((x - rs + P - 1) / P) * P;   // x <= ps < x + P
        if (ps == rs || ps >= re) return;                  // the first piece is the row tile's
        const int pe = min(ps + P, re);
#pragma unroll
        for (int q = 0; q < V; q++) acc[q] = 0.f;
        csr16_piece<T, V, LW>(a, ps, pe, lane, j, acc);
        csr16_carry<V>(a, ps, rs, j, acc);
        return;
    }
    __shared__ float tile[CROW ? 1 : PW][SPMM_CSR16_TILE_ROWS + 1];
    const float alpha = sc.a(), beta = sc.b();
    const int row0 = (int)blockIdx.x * SPMM_CSR16_TILE_ROWS;
#pragma unroll 1
    for (int rr = 0; rr < PER_WARP; rr++) {
        const int rl = warp * PER_WARP + rr, row = row0 + rl;
        float tot[V];
#pragma unroll
        for (int q = 0; q < V; q++) tot[q] = 0.f;
        bool carried = false;
        if (row < a.rows) {                            // warp-uniform
            const int rs = __ldg(a.off + row) - a.base, re = __ldg(a.off + row + 1) - a.base;
            if (a.carry && re - rs > P) {              // split walk: the first piece of a long row to its carry slot
#pragma unroll
                for (int q = 0; q < V; q++) acc[q] = 0.f;
                csr16_piece<T, V, LW>(a, rs, rs + P, lane, j, acc);
                csr16_carry<V>(a, rs, rs, j, acc);
                carried = true;
            } else {
                for (int ps = rs; ps < re; ps += P) {  // tot = 0 + s0 + s1 + ..., the fix-up's order
#pragma unroll
                    for (int q = 0; q < V; q++) acc[q] = 0.f;
                    csr16_piece<T, V, LW>(a, ps, min(ps + P, re), lane, j, acc);
#pragma unroll
                    for (int q = 0; q < V; q++) tot[q] = __fadd_rn(tot[q], acc[q]);
                }
            }
        }
        if constexpr (CROW) {
            if (row < a.rows && !carried) {
#pragma unroll
                for (int q = 0; q < V; q++)
                    if (j + q < a.n) csr16_store<T>(a, true, row, j + q, tot[q], alpha, beta);
            }
        } else {
#pragma unroll
            for (int q = 0; q < V; q++) tile[lane * V + q][rl] = tot[q];
        }
    }
    if constexpr (!CROW) {
        __syncthreads();
        const int row = row0 + lane;
        bool write = row < a.rows;
        if (write && a.carry) write = __ldg(a.off + row + 1) - __ldg(a.off + row) <= P;   // a long row is the fix-up's
        for (int jj = warp; jj < PW; jj += SPMM_CSR16_WARPS) {
            const int c = j0 + jj;
            if (c < a.n && write) csr16_store<T>(a, false, row, c, tile[jj][lane], alpha, beta);
        }
    }
}

// Split walk, part 2: the long row that starts in chunk c (at most one does) gets 0 + s0 + s1 + ... from its carry slots, in
// ascending piece order, written once.  One warp per chunk, 32 columns at a time.
template <typename T>
__global__ void __launch_bounds__(32 * SPMM_CSR16_WARPS) spmm_csr16_fixup_kernel(const SpmmCsr16Args a, const Scalars<float> sc, int c_row) {
    constexpr int P = SPMM_CSR16_PIECE;
    const int lane = (int)threadIdx.x & 31;
    const int c = (int)blockIdx.x * SPMM_CSR16_WARPS + ((int)threadIdx.x >> 5);
    if (c >= a.nchunks) return;
    const long long last = min((long long)(c + 1) * P, (long long)a.nnz) - 1;
    const int r = csr16_row(a, (int)last);
    const int rs = __ldg(a.off + r) - a.base, re = __ldg(a.off + r + 1) - a.base;
    if (rs < c * P || re - rs <= P) return;
    const float alpha = sc.a(), beta = sc.b();
    const int pieces = (re - rs + P - 1) / P;
    for (int j = lane; j < a.n; j += 32) {
        float s = 0.f;
        for (int p = 0; p < pieces; p++) s = __fadd_rn(s, csr16_slot(a, rs + p * P, rs)[j]);
        csr16_store<T>(a, c_row != 0, r, j, s, alpha, beta);
    }
}

// ------------------------------------------------------------------------------------------------ host side
static int csr16_v(int64_t n) { return n <= 32 ? 1 : n <= 64 ? 2 : n <= 128 ? 4 : 8; }
static int64_t csr16_nchunks(int64_t nnz) { return (nnz + SPMM_CSR16_PIECE - 1) / SPMM_CSR16_PIECE; }
// a K-contiguous op(B) is read through a row-major copy in the workspace
static bool csr16_copy(int64_t n, int64_t sbk, int64_t sbj) { return n >= 2 && sbk == 1 && sbj != 1; }
static size_t csr16_copy_bytes(int64_t k, int64_t n) { return ((size_t)k * (size_t)n * 2 + 255) / 256 * 256; }

static int csr16_path(int64_t n, const void* B, int64_t sbk, int64_t sbj) {
    const int v = csr16_v(n);
    if (v == 1 || sbj != 1 || sbk % v || ((uintptr_t)B % (2 * v))) return 1;
    return v;
}

template <typename T, int V, int LW>
static void launch_csr16_main(cudaStream_t st, const dim3& grid, const SpmmCsr16Args& a, const Scalars<float>& sc, bool c_row) {
    if (c_row) spmm_csr16_kernel<T, V, LW, true><<<grid, 32 * SPMM_CSR16_WARPS, 0, st>>>(a, sc);
    else spmm_csr16_kernel<T, V, LW, false><<<grid, 32 * SPMM_CSR16_WARPS, 0, st>>>(a, sc);
}

template <typename T, int V>
static void launch_csr16_v(cudaStream_t st, const dim3& grid, const SpmmCsr16Args& a, const Scalars<float>& sc, bool c_row, int lw) {
    if (V > 1 && lw == V) launch_csr16_main<T, V, V>(st, grid, a, sc, c_row);
    else launch_csr16_main<T, V, 1>(st, grid, a, sc, c_row);
}

template <typename T>
static int launch_csr16(cudaStream_t st, SpmmCsr16Args a, const Scalars<float>& sc, bool c_row, int64_t k, void* copy) {
    if (copy) {                                        // op(B)(k, j) = B[k + j * sbj]: the row-major copy, ld = n
        const dim3 tg((unsigned)((k + 31) / 32), (unsigned)((a.n + 31) / 32));
        spmm_transpose_b_kernel<T><<<tg, 256, 0, st>>>((const T*)a.B, a.sbj, (T*)copy, (int)k, a.n);
        a.B = copy; a.sbk = a.n; a.sbj = 1;
    }
    const int v = csr16_v(a.n), lw = csr16_path(a.n, a.B, a.sbk, a.sbj);
    a.ntiles = (int)((a.rows + SPMM_CSR16_TILE_ROWS - 1) / SPMM_CSR16_TILE_ROWS);
    const bool split = a.carry && a.nnz > SPMM_CSR16_PIECE;   // otherwise no row is long
    if (!split) a.carry = nullptr;
    const long long chunk_ctas = split ? (a.nchunks + SPMM_CSR16_WARPS - 1) / SPMM_CSR16_WARPS : 0;
    const dim3 grid((unsigned)(a.ntiles + chunk_ctas), (unsigned)((a.n + 32 * v - 1) / (32 * v)));
    if (v == 1) launch_csr16_v<T, 1>(st, grid, a, sc, c_row, lw);
    else if (v == 2) launch_csr16_v<T, 2>(st, grid, a, sc, c_row, lw);
    else if (v == 4) launch_csr16_v<T, 4>(st, grid, a, sc, c_row, lw);
    else launch_csr16_v<T, 8>(st, grid, a, sc, c_row, lw);
    if (split)
        spmm_csr16_fixup_kernel<T><<<(unsigned)chunk_ctas, 32 * SPMM_CSR16_WARPS, 0, st>>>(a, sc, c_row);
    return (int)cudaGetLastError();
}

}  // namespace b200

using namespace b200;

extern "C" {

void b200spmm_csr16_params(int32_t* piece, int32_t* lane_entries, int32_t* tile_rows, int32_t* warps, int32_t* max_cols_per_lane) {
    if (piece) *piece = SPMM_CSR16_PIECE;
    if (lane_entries) *lane_entries = SPMM_CSR16_LANE_ENTRIES;
    if (tile_rows) *tile_rows = SPMM_CSR16_TILE_ROWS;
    if (warps) *warps = SPMM_CSR16_WARPS;
    if (max_cols_per_lane) *max_cols_per_lane = SPMM_CSR16_MAX_V;
}

int b200spmm_csr16_path(int64_t n, const void* B, int64_t sbk, int64_t sbj) {
    if (n < 1 || sbk < 0 || sbj < 0) return 0;
    return csr16_path(n, B, sbk, sbj);
}

size_t b200spmm_csr16_workspace_bytes(int64_t k, int64_t n, int64_t nnz, int64_t sbk, int64_t sbj) {
    if (k < 0 || n <= 0 || nnz <= 0) return 0;
    const size_t copy = csr16_copy(n, sbk, sbj) ? csr16_copy_bytes(k, n) : 0;
    return copy + 2 * (size_t)csr16_nchunks(nnz) * (size_t)n * 4;
}

int b200spmm_csr16(void* stream, int ab_type, int c_type, int64_t m, int64_t k, int64_t n, int64_t nnz, const void* offsets,
                   const void* columns, const void* values, int32_t base, const void* alpha, const void* beta, int scalars_on_device,
                   const void* B, int64_t sbk, int64_t sbj, void* C, int64_t ldc, int c_row_major, void* workspace,
                   size_t workspace_bytes) {
    if (ab_type != H16_F16 && ab_type != H16_BF16) return -1;
    if (c_type != ab_type && c_type != H16_F32) return -1;
    if (m < 0 || k < 0 || n < 0 || nnz < 0 || !alpha || !beta || (base != 0 && base != 1)) return -1;
    if (sbk < 0 || sbj < 0) return -1;
    if (m > INT32_MAX - 64 || k > INT32_MAX - 64 || n > 32 * 65535 || nnz > INT32_MAX - 65536) return -1;
    if (nnz > m * k) return -1;
    if (ldc < 1 || ldc < (c_row_major ? n : m)) return -1;
    if (m == 0 || n == 0) return 0;
    if (!C || !offsets || (nnz > 0 && (!columns || !values || !B))) return -1;
    SpmmCsr16Args a;
    a.off = (const int*)offsets; a.col = (const int*)columns; a.val = values; a.B = B; a.C = C; a.carry = nullptr;
    a.sbk = sbk; a.sbj = sbj; a.ldc = ldc;
    a.rows = (int)m; a.n = (int)n; a.nnz = (int)nnz; a.base = base; a.nchunks = (int)csr16_nchunks(nnz); a.ntiles = 0;
    a.c_f32 = c_type == H16_F32;
    Scalars<float> sc;
    if (scalars_on_device) { sc.alpha = 0.f; sc.beta = 0.f; sc.alpha_dev = (const float*)alpha; sc.beta_dev = (const float*)beta; }
    else { sc.alpha = *(const float*)alpha; sc.beta = *(const float*)beta; sc.alpha_dev = nullptr; sc.beta_dev = nullptr; }
    // the workspace holds the row-major copy of a K-contiguous op(B), then the carry slots; a NULL, misaligned or smaller buffer
    // gets neither: the strided gathers and the unsplit walk, with the same bits
    void* copy = nullptr;
    const size_t need = b200spmm_csr16_workspace_bytes(k, n, nnz, sbk, sbj);
    if (need > 0 && workspace && ((uintptr_t)workspace & 15) == 0 && workspace_bytes >= need) {
        const size_t cb = csr16_copy(n, sbk, sbj) ? csr16_copy_bytes(k, n) : 0;
        if (cb) copy = workspace;
        a.carry = (float*)((char*)workspace + cb);
    }
    const cudaStream_t st = (cudaStream_t)stream;
    if (ab_type == H16_F16) return launch_csr16<__half>(st, a, sc, c_row_major != 0, k, copy);
    return launch_csr16<__nv_bfloat16>(st, a, sc, c_row_major != 0, k, copy);
}

}  // extern "C"
