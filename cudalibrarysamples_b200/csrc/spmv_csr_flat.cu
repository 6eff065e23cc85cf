// spmv_csr_flat.cu -- CSR  y = alpha*A*x + beta*y  on H100 (sm_90a) from a "flat" plan built by cusparseSpMV_preprocess.
//
// Why a second CSR path: on skewed matrices (R-MAT) the tile kernels are bound by
// the SM's L1TEX pipe AND by instruction issue, and a third of both goes into finding row boundaries (staged rowOff
// slices, lane-group bookkeeping) and into the shared-memory round trip of every product.  The barrier-free,
// shared-memory-free COO kernel of this library (coo_seg_kernel) ran the same matrix faster than any CSR kernel and
// than the closed library although it streams 4 more bytes per non-zero -- because a warp there only needs
// "which of my 32 elements end a row".  This file gives CSR the same shape:
//
//   preprocess (structure only, integer work, bit-exact against oracle/partition_ref.py::flat_plan):
//     endmask[w]    bit i set  <=>  non-zero 32*w + i is the LAST one of its row             (1 bit per non-zero)
//     chunk_run[c]  number of rows that end before non-zero 256*c (exclusive scan of popcounts)  (4 B per 256 non-zeros)
//     nzrow[j+1]    row index of the j-th non-empty row; nzrow[0] = -1, nzrow[nruns+1] = rows    (4 B per non-empty row)
//   SpMV: csr_flat_kernel -- every warp owns 256 consecutive non-zeros: coalesced 128 B / 256 B loads of col_ind / val,
//     x gathered through L1 (the kernel uses ~100 B of shared memory, so the whole unified L1 serves x: the gather-only
//     rate drops when shared memory is carved out of it, scripts/micro_gather.cu), a step of 32
//     non-zeros inside one row costs one add; a step with row ends costs one butterfly + a segmented shuffle scan with as
//     many levels as its longest remaining segment; the end lanes look their rows up in nzrow and store y.  Rows crossing
//     a warp chunk are stitched per CTA (the last warp to finish, fixed order), rows crossing a CTA (1024 non-zeros) and the
//     EMPTY rows (y = beta*y) by the small csr_flat_fixup_kernel launch that follows: bit-reproducible, no atomics.
//     Three alternatives to that second launch were slower on the GPU this kernel was first tuned on (not re-measured on
//     the H100; scripts/sweep.py FLAT3 and the look-back variants): finishing
//     the CTA-crossing rows inside the kernel (ticketed CTA indices + decoupled look-back, single launch), scaling the empty
//     rows from the chunk that ends the row in front of them, and scaling them by extra CTAs at the end of the main grid.
//
// Replaces cusparse::csrmv_v3_kernel behind cusparseSpMV for preprocessed CSR descriptors (call sites:
// cuSPARSE/spmv_csr/spmv_csr_example.c:104-112, cuSOLVERSp2cuDSS/csreigvsi2cuDSS_double.cpp:148-150,221).
#include "spmv_common.cuh"
#include "config.h"
#include "../../include/b200spmv.h"
#include <vector>

namespace b200 {

#ifndef B200_FLAT_MIN_CTAS
#define B200_FLAT_MIN_CTAS 10     // x 128 threads, 48 registers (swept on an earlier GPU, not re-swept on the H100: scripts/sweep.py FLAT)
#endif
#ifndef B200_FLAT_BATCH        // steps whose col / val loads are all issued before the first gather, fp64 and (unless
#define B200_FLAT_BATCH 4      // B200_FLAT_BATCH32 says otherwise) fp32; swept with the resident CTAs on the H100, DESIGN.md §3.2
#endif
#ifndef B200_FLAT_STEPS
#define B200_FLAT_STEPS 8
#endif
#ifndef B200_FLAT_KBLOOP     // 1: the loop over the batches of a chunk is a run-time loop (code size independent of FLAT_STEPS)
#define B200_FLAT_KBLOOP (B200_FLAT_STEPS > 8)
#endif
#ifndef B200_FLAT_NZPRE      // 1: the chunk's first 32 nzrow entries are loaded with the stream and looked up by shuffle
#define B200_FLAT_NZPRE 0    //    (off: the look-up load hid behind the shuffles on an earlier GPU; not re-measured on the H100)
#endif
constexpr int PLAN_STEPS = 8;                      // the plan's granularity: chunk_run has one entry per 8 steps = 256 non-zeros
constexpr int PLAN_CHUNK = 32 * PLAN_STEPS;
constexpr int FLAT_STEPS = B200_FLAT_STEPS;        // 32-element steps per warp chunk (8, 16 or 32)
constexpr int FLAT_CHUNK = 32 * FLAT_STEPS;        // non-zeros per warp
static_assert(FLAT_STEPS % PLAN_STEPS == 0 && FLAT_STEPS <= 32, "a warp chunk is 1, 2 or 4 plan chunks");
#ifndef B200_FLAT_WARPS
#define B200_FLAT_WARPS 4
#endif
constexpr int FLAT_WARPS = B200_FLAT_WARPS;         // warp chunks stitched per CTA (a divisor of 8)
constexpr int FLAT_BLOCK = 32 * FLAT_WARPS;
constexpr int FLAT_CTA_NNZ = FLAT_CHUNK * FLAT_WARPS;   // 2048 non-zeros per CTA
constexpr int FLAT_CTA_WORDS = FLAT_CTA_NNZ / 32;
constexpr int FLAT_PAD_NNZ = 2048;                 // the plan arrays are padded to this many non-zeros (independent of FLAT_WARPS)
static_assert(FLAT_PAD_NNZ % FLAT_CTA_NNZ == 0, "FLAT_WARPS x FLAT_STEPS must divide 64");
constexpr int FLAT_BATCH64 = B200_FLAT_BATCH;
#ifdef B200_FLAT_BATCH32
constexpr int FLAT_BATCH32 = B200_FLAT_BATCH32;
#else
constexpr int FLAT_BATCH32 = B200_FLAT_BATCH;      // fp32 too: a batch of 4 ran fp32 R-MAT 1 M 6 % faster than 8 on the H100 (DESIGN.md §3.2)
#endif
constexpr int SCAN_ITEMS = 2048;                   // items per block of the preprocessing scans
#ifndef B200_FLAT_FIXUP_AHEAD
#define B200_FLAT_FIXUP_AHEAD 8                    // CTA partials csr_flat_fixup_kernel loads per round trip
#endif
constexpr int FIXUP_AHEAD = B200_FLAT_FIXUP_AHEAD;
static_assert(FLAT_STEPS % FLAT_BATCH64 == 0 && FLAT_STEPS % FLAT_BATCH32 == 0, "steps per chunk must be a multiple of the batch");

// Hot columns of x.  Preprocess picks the most-used columns whose values fit B200_FLAT_HOT_BYTES, and every SpMV first packs
// their x values densely (xh) so the gather of csr_flat_kernel finds them on fewer, fully used cache lines.  On R-MAT the
// hot columns are scattered over lines shared with cold columns; packed, more of the gathers hit L1.  With a hot plan the
// cold gathers go to L2 only (ldg_cold, spmv_common.cuh): when they allocated L1 lines, their stream (about half the
// gathers of R-MAT 1 M, nearly all on distinct lines) evicted packed lines before their next use, so a budget beyond 64 KB
// bought pack traffic and no hits.  With the cold gathers out of L1, budgets up to about 128 KB gain.
#ifndef B200_FLAT_HOT_BYTES
#define B200_FLAT_HOT_BYTES (128 * 1024)  // swept over 0 ... 192 KB with each cold-gather policy on the H100: scripts/sweep.py flat_l1
#endif
constexpr int HOT_BYTES = B200_FLAT_HOT_BYTES;
constexpr int HOT_MAX = HOT_BYTES / 4;              // slots of the hot list: fp32 fits twice as many values as fp64
constexpr int HOT_MIN_PERMILLE = 200;               // the hot columns must take at least this share of nnz, else no hot plan
constexpr int HOT_BINS = 1 << 16;                   // column-count histogram: bin n = columns used n times, the last bin >= n
static_assert(HOT_BYTES % 8 == 0, "B200_FLAT_HOT_BYTES must be a multiple of 8");

struct FlatPlan {
    unsigned* endmask;    // [nctas * 64]   zero-padded behind nnz
    int*      chunk_run;  // [nctas * 8 + 1]
    int*      nzrow;      // [rows + 2]
    double*   cta_first;  // [nctas]  sum in front of the CTA's first row end (whole CTA if no row ends in it)
    double*   cta_last;   // [nctas]  sum behind the CTA's last row end
    int*      cta_flags;  // [nctas]  1: at least one row ends in this CTA
    int*      ctl;        // [0] nruns (non-empty rows), [1] steps without a row end, [2] steps, [4] hot columns H, [5] threshold,
                          // [6..7] non-zeros in columns of the last histogram bin (uint64)
    int*      scratch;    // block sums of the scans
    int*      colp;       // [nchunks * 256]  ~j for hot slot j, else the 0-based column; 0 behind nnz.  Column counts before that.
    int*      hot;        // [HOT_MAX]        0-based columns of the hot slots, ascending
    void*     xh;         // [HOT_BYTES]      x[hot[j]], refreshed by every SpMV with H > 0
    unsigned* bins;       // [HOT_BINS]
};

static inline int64_t flat_num_ctas(int64_t nnz) { return (nnz + FLAT_CTA_NNZ - 1) / FLAT_CTA_NNZ; }
static inline int64_t flat_num_chunks_padded(int64_t nnz) { return (nnz + FLAT_PAD_NNZ - 1) / FLAT_PAD_NNZ * (FLAT_PAD_NNZ / PLAN_CHUNK); }

static size_t flat_layout(int64_t rows, int64_t nnz, void* ws, FlatPlan* p) {
    const size_t nchunks = (size_t)flat_num_chunks_padded(nnz);
    const size_t nctas = nchunks;                                  // upper bound for every FLAT_WARPS (one CTA per chunk)
    const size_t ncolp = HOT_BYTES > 0 ? nchunks * PLAN_CHUNK : 0; // also the largest column count the hot plan takes
    const int64_t nscan_items = rows > (int64_t)ncolp ? rows : (int64_t)ncolp;
    const size_t nscan = (size_t)((nscan_items > (int64_t)nchunks ? nscan_items : (int64_t)nchunks) / SCAN_ITEMS + 2);
    size_t o = 0;
    const size_t o_mask = o;  o = round_up_256(o + nchunks * PLAN_STEPS * sizeof(unsigned));
    const size_t o_crun = o;  o = round_up_256(o + (nchunks + 1) * sizeof(int));
    const size_t o_nzr  = o;  o = round_up_256(o + ((size_t)rows + 2 + 32) * sizeof(int));   // + 32: the kernel's look-ahead window
    const size_t o_cf   = o;  o = round_up_256(o + nctas * sizeof(double));
    const size_t o_cl   = o;  o = round_up_256(o + nctas * sizeof(double));
    const size_t o_fl   = o;  o = round_up_256(o + nctas * sizeof(int));
    const size_t o_ctl  = o;  o = round_up_256(o + 64);
    const size_t o_scr  = o;  o = round_up_256(o + nscan * sizeof(int));
    const bool   hot = ncolp > 0;
    const size_t o_colp = o;  o = round_up_256(o + ncolp * sizeof(int));
    const size_t o_hot  = o;  o = round_up_256(o + (hot ? HOT_MAX * sizeof(int) : 0));
    const size_t o_xh   = o;  o = round_up_256(o + (hot ? HOT_BYTES : 0));
    const size_t o_bins = o;  o = round_up_256(o + (hot ? HOT_BINS * sizeof(unsigned) : 0));
    if (p) {
        char* b = (char*)ws;
        p->endmask = (unsigned*)(b + o_mask); p->chunk_run = (int*)(b + o_crun); p->nzrow = (int*)(b + o_nzr);
        p->cta_first = (double*)(b + o_cf); p->cta_last = (double*)(b + o_cl); p->cta_flags = (int*)(b + o_fl);
        p->ctl = (int*)(b + o_ctl); p->scratch = (int*)(b + o_scr);
        p->colp = (int*)(b + o_colp); p->hot = (int*)(b + o_hot); p->xh = (void*)(b + o_xh); p->bins = (unsigned*)(b + o_bins);
    }
    return o;
}

// ------------------------------------------------------------------------------------------------
// preprocess
// ------------------------------------------------------------------------------------------------
__global__ void flat_mark_ends_kernel(const int* __restrict__ off, int base, int64_t rows, unsigned* __restrict__ endmask) {
    for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < rows; r += (int64_t)gridDim.x * blockDim.x) {
        const int b = off[r] - base, e = off[r + 1] - base;
        if (e > b) atomicOr(endmask + ((e - 1) >> 5), 1u << ((e - 1) & 31));
    }
}

// value functors of the two scans
struct RowNonEmpty {
    const int* off;
    __device__ __forceinline__ int operator()(int64_t r) const { return off[r + 1] > off[r] ? 1 : 0; }
};
struct ChunkEnds {
    const unsigned* endmask;
    __device__ __forceinline__ int operator()(int64_t c) const {
        int n = 0;
#pragma unroll
        for (int k = 0; k < PLAN_STEPS; k++) n += __popc(endmask[c * PLAN_STEPS + k]);
        return n;
    }
};

// exclusive prefix sum in three launches: block sums, one block scans them, blocks scan locally and emit
template <typename V>
__global__ void __launch_bounds__(256) scan_block_sums_kernel(V value, int64_t n, int* __restrict__ block_sums) {
    __shared__ int sw[8];
    const int64_t i0 = (int64_t)blockIdx.x * SCAN_ITEMS;
    int s = 0;
    for (int k = threadIdx.x; k < SCAN_ITEMS; k += 256) {
        const int64_t i = i0 + k;
        s += i < n ? value(i) : 0;
    }
    s = warp_allsum(s);
    if ((threadIdx.x & 31) == 0) sw[threadIdx.x >> 5] = s;
    __syncthreads();
    if (threadIdx.x == 0) {
        int t = 0;
#pragma unroll
        for (int w = 0; w < 8; w++) t += sw[w];
        block_sums[blockIdx.x] = t;
    }
}

__global__ void __launch_bounds__(1024) scan_of_block_sums_kernel(int* __restrict__ block_sums, int64_t nb, int* __restrict__ total) {
    __shared__ int sw[32];
    __shared__ int carry;
    if (threadIdx.x == 0) carry = 0;
    __syncthreads();
    for (int64_t i0 = 0; i0 < nb; i0 += 1024) {
        const int64_t i = i0 + threadIdx.x;
        const int v = i < nb ? block_sums[i] : 0;
        int incl = v;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) { const int t = __shfl_up_sync(0xffffffffu, incl, o); if ((threadIdx.x & 31) >= o) incl += t; }
        if ((threadIdx.x & 31) == 31) sw[threadIdx.x >> 5] = incl;
        __syncthreads();
        if (threadIdx.x < 32) {
            const int w = sw[threadIdx.x];
            int wi = w;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) { const int t = __shfl_up_sync(0xffffffffu, wi, o); if (threadIdx.x >= o) wi += t; }
            sw[threadIdx.x] = wi - w;                   // exclusive prefix of the warp sums
        }
        __syncthreads();
        const int excl = carry + sw[threadIdx.x >> 5] + incl - v;
        if (i < nb) block_sums[i] = excl;
        __syncthreads();
        if (threadIdx.x == 1023) carry = excl + v;
        __syncthreads();
    }
    if (threadIdx.x == 0) *total = carry;
}

template <typename V, typename E>
__global__ void __launch_bounds__(256) scan_emit_kernel(V value, E emit, int64_t n, const int* __restrict__ block_sums) {
    __shared__ int sw[8];
    __shared__ int carry;
    if (threadIdx.x == 0) carry = block_sums[blockIdx.x];
    __syncthreads();
    const int64_t i0 = (int64_t)blockIdx.x * SCAN_ITEMS;
    for (int k0 = 0; k0 < SCAN_ITEMS; k0 += 256) {
        const int64_t i = i0 + k0 + threadIdx.x;
        const int v = i < n ? value(i) : 0;
        int incl = v;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) { const int t = __shfl_up_sync(0xffffffffu, incl, o); if ((threadIdx.x & 31) >= o) incl += t; }
        if ((threadIdx.x & 31) == 31) sw[threadIdx.x >> 5] = incl;
        __syncthreads();
        int woff = 0;
#pragma unroll
        for (int w = 0; w < 8; w++) woff += w < (int)(threadIdx.x >> 5) ? sw[w] : 0;
        const int excl = carry + woff + incl - v;
        if (i < n) emit(i, excl, v);
        __syncthreads();
        if (threadIdx.x == 255) carry = excl + v;
        __syncthreads();
    }
}

struct EmitNzRow {
    int* nzrow;
    __device__ __forceinline__ void operator()(int64_t r, int rank, int v) const { if (v) nzrow[rank + 1] = (int)r; }
};
struct EmitChunkRun {
    int* chunk_run;
    __device__ __forceinline__ void operator()(int64_t c, int before, int) const { chunk_run[c] = before; }
};

__global__ void flat_finish_kernel(FlatPlan p, int64_t rows, int64_t nchunks, int64_t nwords) {
    // nzrow sentinels, the closing chunk_run entry, and the statistic the shim uses to pick the kernel
    const int nruns = p.ctl[0];
    if (blockIdx.x == 0 && threadIdx.x == 0) {
        p.nzrow[0] = -1;
        p.nzrow[nruns + 1] = (int)rows;
        p.chunk_run[nchunks] = nruns;
        p.ctl[2] = (int)nwords;
    }
    int quiet = 0;
    for (int64_t w = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; w < nwords; w += (int64_t)gridDim.x * blockDim.x)
        quiet += p.endmask[w] == 0u;
    quiet = warp_allsum(quiet);
    if ((threadIdx.x & 31) == 0 && quiet) atomicAdd(p.ctl + 1, quiet);
}

// hot plan: uses per column (colp doubles as the counter array), then how many columns have each use count
__global__ void flat_hot_count_kernel(const int* __restrict__ col, int base, int64_t nnz, int64_t cols, int* __restrict__ cnt) {
    for (int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; k < nnz; k += (int64_t)gridDim.x * blockDim.x) {
        const int64_t c = (int64_t)__ldg(col + k) - base;
        if (c >= 0 && c < cols) atomicAdd(cnt + c, 1);
    }
}

__global__ void flat_hot_bins_kernel(const int* __restrict__ cnt, int64_t cols, unsigned* __restrict__ bins,
                                     unsigned long long* __restrict__ last_bin_nnz) {
    for (int64_t c = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; c < cols; c += (int64_t)gridDim.x * blockDim.x) {
        const int n = cnt[c];
        if (n < 2) continue;
        atomicAdd(bins + min(n, HOT_BINS - 1), 1u);
        if (n >= HOT_BINS - 1) atomicAdd(last_bin_nnz, (unsigned long long)n);
    }
}

struct HotFlag {
    const int* cnt;
    int        tau;
    __device__ __forceinline__ int operator()(int64_t c) const { return cnt[c] >= tau ? 1 : 0; }
};
struct EmitHot {
    int* hot;
    __device__ __forceinline__ void operator()(int64_t c, int rank, int v) const { if (v) hot[rank] = (int)c; }
};

// colp[k] = ~j if column col[k] - base is hot slot j (binary search of the ascending hot list), else col[k] - base
__global__ void flat_hot_colp_kernel(const int* __restrict__ col, int base, int64_t nnz, int64_t npad, const int* __restrict__ hot,
                                     int nhot, int tau, int* __restrict__ colp, int* __restrict__ ctl) {
    if (blockIdx.x == 0 && threadIdx.x == 0) { ctl[4] = nhot; ctl[5] = tau; }
    for (int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; k < npad; k += (int64_t)gridDim.x * blockDim.x) {
        int v = 0;                                          // behind nnz: a column that is never hot
        if (k < nnz) {
            v = __ldg(col + k) - base;
            int lo = 0, hi = nhot;
            while (lo < hi) {
                const int mid = (lo + hi) >> 1;
                if (__ldg(hot + mid) < v) lo = mid + 1; else hi = mid;
            }
            if (lo < nhot && __ldg(hot + lo) == v) v = ~lo;
        }
        colp[k] = v;
    }
}

// The threshold: the smallest tau >= 2 whose columns (used >= tau times) fit `slots`; no hot plan (0) when even the last bin does
// not fit or the hot columns take less than HOT_MIN_PERMILLE of nnz.
static int flat_hot_choose(const unsigned* bins, unsigned long long last_bin_nnz, int64_t nnz, int64_t slots, int* tau_out) {
    long long h = 0, covered = (long long)last_bin_nnz;
    int tau = 0;
    for (int t = HOT_BINS - 1; t >= 2; t--) {
        if (h + bins[t] > slots) break;
        h += bins[t];
        if (t < HOT_BINS - 1) covered += (long long)t * bins[t];
        tau = t;
    }
    *tau_out = tau;
    if (tau == 0 || h == 0 || covered * 1000 < (long long)HOT_MIN_PERMILLE * nnz) return 0;
    return (int)h;
}

// ------------------------------------------------------------------------------------------------
// SpMV
// ------------------------------------------------------------------------------------------------
template <typename T>
struct FlatArgs {
    const int* off;
    const int* col;       // the caller's col_ind, or colp of a hot plan (then base == 0)
    const T*   val;
    const T*   x;
    const T*   xh;        // packed hot values: read for col < 0
    T*         y;
    int        base;
    int        rows;
    int        nnz;
    Scalars<T> s;
    FlatPlan   plan;
};

// y[r] = alpha * v + beta * y[r]; beta == 0 never reads y (predicated load, no branch)
template <typename T>
__device__ __forceinline__ void flat_store_y(T* yp, T alpha, T v, T beta) {
    T old = T(0);
    if (beta != T(0)) old = *yp;
    *yp = alpha * v + beta * old;
}

// HOT: the matrix has a hot plan (col is colp).  Only then do the cold gathers take the ldg_cold policy: without packed hot
// lines to protect, every gather is "cold", and keeping them all out of L1 loses every L1 hit (DESIGN.md §3.2, 0 KB row).
template <typename T, bool HOT>
__global__ void __launch_bounds__(FLAT_BLOCK, B200_FLAT_MIN_CTAS) csr_flat_kernel(const FlatArgs<T> a) {
    __shared__ T   sFirst[FLAT_WARPS], sLast[FLAT_WARPS];
    __shared__ int sFrow[FLAT_WARPS];                      // >= 0: row of the chunk's first row end (deferred to the stitch)
    __shared__ int sArrived;                               // warps that have deposited their partials
    if (threadIdx.x == 0) sArrived = 0;
    __syncthreads();                                       // the only CTA-wide barrier, before any work: nobody waits at the end

    const int lane = (int)threadIdx.x & 31, warp = (int)threadIdx.x >> 5;
    const long long c = (long long)blockIdx.x * FLAT_WARPS + warp;      // warp chunk
    const long long c0 = c * FLAT_CHUNK;
    const bool active = c0 < a.nnz;
    const T alpha = a.s.a(), beta = a.s.b();
    T   acc = T(0), first = T(0), last = T(0);
    int frow = -1;

    if (active) {
        const int n0 = (int)c0, n1 = min(n0 + FLAT_CHUNK, a.nnz);
        const unsigned mreg = lane < FLAT_STEPS ? __ldg(a.plan.endmask + c * FLAT_STEPS + lane) : 0u;
        int run = __ldg(a.plan.chunk_run + c * (FLAT_STEPS / PLAN_STEPS));   // rows that ended before this chunk
#if B200_FLAT_NZPRE
        const int run0 = run;
        const int nzw = __ldg(a.plan.nzrow + run0 + 1 + lane);              // rows of the chunk's first 32 row ends
#endif
        const int* colp = a.col + n0;
        const T*   valp = a.val + n0;
        const T*   xp = a.x - a.base;
        constexpr int FLAT_BATCH = sizeof(T) == 8 ? FLAT_BATCH64 : FLAT_BATCH32;
        int cc[FLAT_BATCH];
        T   vv[FLAT_BATCH];
        auto issue = [&](int kb) {
#pragma unroll
            for (int k = 0; k < FLAT_BATCH; k++) {
                const int e = (kb + k) * 32 + lane;
                const bool live = n0 + e < n1;
                cc[k] = live ? ldg_stream(colp + e) : a.base;
                vv[k] = live ? ldg_stream(valp + e) : T(0);
            }
        };
        issue(0);
        // Unrolled over the 8 steps (static register indexing, no loop control), but the scan inside a flush is a run-time
        // loop: with everything unrolled the kernel outgrows the instruction cache and stalls on instruction fetch; with
        // run-time step loops most of what it executes is select chains / loop control.
#if B200_FLAT_KBLOOP
#pragma unroll 1
#else
#pragma unroll
#endif
        for (int kb = 0; kb < FLAT_STEPS; kb += FLAT_BATCH) {
            if (n0 + kb * 32 >= n1) break;                 // warp-uniform: the matrix' last chunk may be short
            T p[FLAT_BATCH];
#pragma unroll
            for (int k = 0; k < FLAT_BATCH; k++)
                p[k] = (n0 + (kb + k) * 32 + lane < n1)
                           ? vv[k] * (HOT && cc[k] < 0 ? __ldg(a.xh + ~cc[k]) : HOT ? ldg_cold(xp + cc[k]) : __ldg(xp + cc[k]))
                           : T(0);
            if (kb + FLAT_BATCH < FLAT_STEPS && n0 + (kb + FLAT_BATCH) * 32 < n1) issue(kb + FLAT_BATCH);
#pragma unroll
            for (int k = 0; k < FLAT_BATCH; k++) {
                const unsigned m = __shfl_sync(0xffffffffu, mreg, kb + k);
                const T pk = p[k];
                if (m == 0u) { acc += pk; continue; }      // the whole step lies inside one row
                const int e1 = __ffs(m) - 1, ek = 31 - __clz(m);
                // my row (if I end one): issued first, the look-up's latency hides behind the shuffles below
                const bool is_end = (m >> lane) & 1u;
                int row = 0;
#if B200_FLAT_NZPRE
                {
                    const int j = run - run0 + __popc(m & ((1u << lane) - 1u));     // my row end is the chunk's j-th
                    row = __shfl_sync(0xffffffffu, nzw, j & 31);
                    if (is_end && j >= 32) row = __ldg(a.plan.nzrow + run0 + j + 1); // more than 32 rows end in this chunk
                }
#else
                if (is_end) row = __ldg(a.plan.nzrow + run + __popc(m & ((1u << lane) - 1u)) + 1);   // (run + k)-th non-empty row
#endif
                const T t1 = warp_allsum(acc + (lane <= e1 ? pk : T(0)));
                T q = (lane > e1 && lane <= ek) ? pk : T(0);
                if (m & (m - 1u)) {                        // more rows end: segmented inclusive scan
                    const unsigned below = m & ((1u << lane) - 1u);
                    const int dist = (lane > e1 && lane <= ek) ? lane - (32 - __clz(below)) : 0;
#pragma unroll 1
                    for (int d = 1; d < 32; d <<= 1) {
                        if (__ballot_sync(0xffffffffu, dist >= d) == 0u) break;
                        const T t = __shfl_up_sync(0xffffffffu, q, d);
                        if (dist >= d) q += t;
                    }
                }
                const T res = lane == e1 ? t1 : q;
                bool mine = is_end;
                if (frow < 0) {                            // the chunk's first row end goes to the stitch
                    first = __shfl_sync(0xffffffffu, res, e1);
                    frow = __shfl_sync(0xffffffffu, row, e1);
                    mine = is_end && lane != e1;
                }
                if (mine) flat_store_y(a.y + row, alpha, res, beta);
                run += __popc(m);
                acc = lane > ek ? pk : T(0);
            }
        }
        // non-zeros behind the chunk's last row end belong to a row that continues in the next chunk
        const int  el = n1 - 1 - n0;                       // the chunk's last live element
        const unsigned ml = __shfl_sync(0xffffffffu, mreg, el >> 5);
        if (!((ml >> (el & 31)) & 1u)) last = warp_allsum(acc);
    }
    // The warp that deposits its partials LAST stitches the CTA (fixed warp order -> bit-reproducible); the others are gone.
    int arrived = 0;
    if (lane == 0) {
        if (frow >= 0) { sFirst[warp] = first; sLast[warp] = last; }
        else           { sFirst[warp] = last;  sLast[warp] = T(0); }     // no row ended here: the whole chunk is one partial
        sFrow[warp] = frow;
        __threadfence_block();
        arrived = atomicAdd(&sArrived, 1);
    }
    if (lane == 0 && arrived == FLAT_WARPS - 1) {
        __threadfence_block();
        const long long cta = blockIdx.x;
        const bool starts_row = cta == 0 || (__ldg(a.plan.endmask + cta * FLAT_CTA_WORDS - 1) >> 31);   // a row starts with this CTA
        T    running = T(0);
        bool has = false;
#pragma unroll
        for (int w = 0; w < FLAT_WARPS; w++) {
            const int fr = sFrow[w];
            if (fr >= 0) {
                const T tot = running + sFirst[w];
                if (!has && !starts_row) a.plan.cta_first[cta] = (double)tot;            // the row began in an earlier CTA
                else flat_store_y(a.y + fr, alpha, tot, beta);
                running = sLast[w];
                has = true;
            } else {
                running += sFirst[w];
            }
        }
        if (!has) { a.plan.cta_first[cta] = (double)running; a.plan.cta_last[cta] = 0.0; }
        else      a.plan.cta_last[cta] = (double)running;
        a.plan.cta_flags[cta] = has ? 1 : 0;
    }
}

// Second (small) launch: (1) rows that cross CTA borders -- thread t owns the row that STARTS in CTA t and runs past its
// end, partials added in CTA order; (2) EMPTY rows, which the main kernel never sees: y = beta * y, one thread per row.
template <typename T>
__global__ void __launch_bounds__(256) csr_flat_fixup_kernel(const FlatArgs<T> a, long long nctas) {
    const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const T alpha = a.s.a(), beta = a.s.b();
    if (t < a.rows && beta != T(1)) {                       // beta == 1 (a later column panel of a sharded product): y stays as it is
        if (__ldg(a.off + t) == __ldg(a.off + t + 1)) flat_store_y(a.y + t, alpha, T(0), beta);
    }
    if (t >= nctas - 1) return;
    const bool tail_open = !(__ldg(a.plan.endmask + (t + 1) * FLAT_CTA_WORDS - 1) >> 31);
    if (!tail_open) return;
    const bool has = __ldcg(a.plan.cta_flags + t) != 0;
    const bool starts_row = t == 0 || (__ldg(a.plan.endmask + t * FLAT_CTA_WORDS - 1) >> 31);
    if (!has && !starts_row) return;                       // CTA t lies inside a row that started earlier
    double sum = has ? __ldcg(a.plan.cta_last + t) : __ldcg(a.plan.cta_first + t);
    // Add cta_first of the CTAs the row runs through, up to the one it ends in (cta_flags != 0), in CTA order.  The heaviest
    // rows of a skewed matrix cross dozens of CTAs: FIXUP_AHEAD CTAs are loaded per L2 round trip instead of one after the
    // other.  The last CTA always ends a row, so clamping the look-ahead to it changes no sum.
    long long u = t + 1;
    for (bool done = false; !done; ) {
        int    fl[FIXUP_AHEAD];
        double fs[FIXUP_AHEAD];
#pragma unroll
        for (int k = 0; k < FIXUP_AHEAD; k++) {
            const long long v = min(u + k, nctas - 1);
            fl[k] = __ldcg(a.plan.cta_flags + v);
            fs[k] = __ldcg(a.plan.cta_first + v);
        }
#pragma unroll
        for (int k = 0; k < FIXUP_AHEAD; k++) {
            if (done) continue;
            sum += fs[k];
            if (fl[k] != 0) { done = true; u += k; }
        }
        if (!done) u += FIXUP_AHEAD;
    }
    const int row = __ldg(a.plan.nzrow + __ldg(a.plan.chunk_run + u * (FLAT_CTA_NNZ / PLAN_CHUNK)) + 1);
    flat_store_y(a.y + row, alpha, (T)sum, beta);
}

template <typename T>
__global__ void flat_scale_y_kernel(T* __restrict__ y, int64_t rows, Scalars<T> s) {
    const T beta = s.b();
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < rows; i += (int64_t)gridDim.x * blockDim.x)
        y[i] = beta == T(0) ? T(0) : beta * y[i];
}

template <typename T>
__global__ void flat_hot_pack_kernel(const int* __restrict__ hot, int nhot, const T* __restrict__ x, T* __restrict__ xh) {
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j < nhot) xh[j] = __ldg(x + __ldg(hot + j));
}

template <typename T>
static int launch_flat(cudaStream_t stream, int64_t rows, int64_t nnz, const void* off, const void* col, const void* val, int base,
                       const void* alpha, const void* beta, int on_device, const void* x, void* y, void* ws, int nhot) {
    if (nhot < 0 || (int64_t)nhot * (int64_t)sizeof(T) > HOT_BYTES || (nhot > 0 && nnz == 0)) return -1;
    FlatArgs<T> a;
    a.off = (const int*)off; a.col = (const int*)col; a.val = (const T*)val; a.x = (const T*)x; a.y = (T*)y;
    a.base = base; a.rows = (int)rows; a.nnz = (int)nnz;
    set_scalars(a.s, alpha, beta, on_device);
    flat_layout(rows, nnz, ws, &a.plan);
    a.xh = (const T*)a.plan.xh;
    stats().last_csr_kernel = sizeof(T) == 8 ? "b200::csr_flat_kernel<double>" : "b200::csr_flat_kernel<float>";
    if (nnz == 0) {
        int64_t blocks = (rows + 255) / 256;
        if (blocks > 132 * 16) blocks = 132 * 16;
        flat_scale_y_kernel<T><<<(unsigned)blocks, 256, 0, stream>>>((T*)y, rows, a.s);
        return (int)cudaGetLastError();
    }
    if (nhot > 0) {                                         // same products in the same order: only where x[c] is read from changes
        flat_hot_pack_kernel<T><<<(unsigned)((nhot + 255) / 256), 256, 0, stream>>>(a.plan.hot, nhot, (const T*)x, (T*)a.plan.xh);
        a.col = a.plan.colp;
        a.base = 0;
    }
    const int64_t nctas = flat_num_ctas(nnz);
    if (nhot > 0) csr_flat_kernel<T, true><<<(unsigned)nctas, FLAT_BLOCK, 0, stream>>>(a);
    else          csr_flat_kernel<T, false><<<(unsigned)nctas, FLAT_BLOCK, 0, stream>>>(a);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return (int)e;
    // empty rows + CTA-crossing rows; with a host-side beta == 1 the empty rows need no pass at all
    const bool skip_rows = !on_device && *(const T*)beta == T(1);
    const int64_t work = (!skip_rows && rows > nctas - 1) ? rows : (nctas - 1 > 0 ? nctas - 1 : 1);
    csr_flat_fixup_kernel<T><<<(unsigned)((work + 255) / 256), 256, 0, stream>>>(a, (long long)nctas);
    return (int)cudaGetLastError();
}

}  // namespace b200

using namespace b200;

extern "C" {

size_t b200spmv_csr_flat_workspace_bytes(int64_t rows, int64_t nnz) {
    if (rows < 0 || nnz < 0) return 0;
    return flat_layout(rows, nnz, nullptr, nullptr);
}

int b200spmv_csr_flat_analyze(void* stream_, int64_t rows, int64_t nnz, const void* row_offsets, int32_t base, void* workspace) {
    if (rows < 0 || nnz < 0 || rows > INT32_MAX - 2 || nnz > INT32_MAX - 65536 || !workspace || (rows > 0 && !row_offsets)) return -1;
    cudaStream_t stream = (cudaStream_t)stream_;
    FlatPlan p;
    const size_t total = flat_layout(rows, nnz, workspace, &p);
    (void)total;
    const int64_t nchunks = flat_num_chunks_padded(nnz), nwords = (nnz + 31) / 32;
    cudaError_t e = cudaMemsetAsync(p.endmask, 0, (size_t)nchunks * PLAN_STEPS * sizeof(unsigned), stream);
    if (e != cudaSuccess) return (int)e;
    e = cudaMemsetAsync(p.ctl, 0, 64, stream);
    if (e != cudaSuccess) return (int)e;
    const int* off = (const int*)row_offsets;
    if (rows > 0) {
        int64_t blocks = (rows + 255) / 256;
        if (blocks > 132 * 32) blocks = 132 * 32;
        flat_mark_ends_kernel<<<(unsigned)blocks, 256, 0, stream>>>(off, base, rows, p.endmask);
        // rank of every non-empty row -> nzrow
        const int64_t nb = (rows + SCAN_ITEMS - 1) / SCAN_ITEMS;
        RowNonEmpty v{off};
        scan_block_sums_kernel<<<(unsigned)nb, 256, 0, stream>>>(v, rows, p.scratch);
        scan_of_block_sums_kernel<<<1, 1024, 0, stream>>>(p.scratch, nb, p.ctl);            // ctl[0] = nruns
        scan_emit_kernel<<<(unsigned)nb, 256, 0, stream>>>(v, EmitNzRow{p.nzrow}, rows, p.scratch);
    }
    if (nchunks > 0) {
        const int64_t nb = (nchunks + SCAN_ITEMS - 1) / SCAN_ITEMS;
        ChunkEnds v{p.endmask};
        scan_block_sums_kernel<<<(unsigned)nb, 256, 0, stream>>>(v, nchunks, p.scratch);
        scan_of_block_sums_kernel<<<1, 1024, 0, stream>>>(p.scratch, nb, p.ctl + 3);          // ctl[3] = nruns again (check)
        scan_emit_kernel<<<(unsigned)nb, 256, 0, stream>>>(v, EmitChunkRun{p.chunk_run}, nchunks, p.scratch);
    }
    int64_t fb = (nwords + 255) / 256;
    if (fb > 132 * 8) fb = 132 * 8;
    if (fb < 1) fb = 1;
    flat_finish_kernel<<<(unsigned)fb, 256, 0, stream>>>(p, rows, nchunks, nwords);
    return (int)cudaGetLastError();
}

// byte offsets of the plan arrays inside the workspace (parity tests read them back and compare bit for bit)
void b200spmv_csr_flat_plan_offsets(int64_t rows, int64_t nnz, size_t* endmask, size_t* chunk_run, size_t* nzrow, size_t* ctl) {
    FlatPlan p;
    flat_layout(rows, nnz, nullptr, &p);
    if (endmask) *endmask = (size_t)((char*)p.endmask - (char*)nullptr);
    if (chunk_run) *chunk_run = (size_t)((char*)p.chunk_run - (char*)nullptr);
    if (nzrow) *nzrow = (size_t)((char*)p.nzrow - (char*)nullptr);
    if (ctl) *ctl = (size_t)((char*)p.ctl - (char*)nullptr);
}

void b200spmv_csr_flat_params(int32_t* warp_chunk, int32_t* cta_nnz, int32_t* plan_chunk) {
    if (warp_chunk) *warp_chunk = FLAT_CHUNK;
    if (cta_nnz) *cta_nnz = FLAT_CTA_NNZ;
    if (plan_chunk) *plan_chunk = PLAN_CHUNK;
}

int b200spmv_csr_flat_hot_analyze(void* stream_, int dtype, int64_t rows, int64_t cols, int64_t nnz, const void* col_ind, int32_t base,
                                  void* workspace, int32_t* hot_out) {
    if (!hot_out) return -1;
    *hot_out = 0;
    if (rows < 0 || cols < 0 || nnz < 0 || rows > INT32_MAX - 2 || cols > INT32_MAX || nnz > INT32_MAX - 65536 || !workspace ||
        (nnz > 0 && !col_ind) || (dtype != 0 && dtype != 1))
        return -1;
    cudaStream_t stream = (cudaStream_t)stream_;
    FlatPlan p;
    flat_layout(rows, nnz, workspace, &p);
    cudaError_t e = cudaMemsetAsync(p.ctl + 4, 0, 4 * sizeof(int), stream);
    if (e != cudaSuccess) return (int)e;
    const int64_t npad = flat_num_chunks_padded(nnz) * PLAN_CHUNK;
    cudaStreamCaptureStatus cap = cudaStreamCaptureStatusNone;
    if (cudaStreamIsCapturing(stream, &cap) != cudaSuccess) cap = cudaStreamCaptureStatusNone;
    // the counters live in colp: no hot plan for more columns than that holds, nor under capture (the threshold is read back)
    if (HOT_BYTES == 0 || nnz == 0 || cols > npad || cap != cudaStreamCaptureStatusNone) return 0;
    const int* col = (const int*)col_ind;
    unsigned long long* last_bin_nnz = (unsigned long long*)(p.ctl + 6);
    if ((e = cudaMemsetAsync(p.colp, 0, (size_t)cols * sizeof(int), stream)) != cudaSuccess) return (int)e;
    if ((e = cudaMemsetAsync(p.bins, 0, HOT_BINS * sizeof(unsigned), stream)) != cudaSuccess) return (int)e;
    int64_t blocks = (nnz + 255) / 256;
    if (blocks > 132 * 32) blocks = 132 * 32;
    flat_hot_count_kernel<<<(unsigned)blocks, 256, 0, stream>>>(col, base, nnz, cols, p.colp);
    int64_t cblocks = (cols + 255) / 256;
    if (cblocks > 132 * 32) cblocks = 132 * 32;
    if (cblocks < 1) cblocks = 1;
    flat_hot_bins_kernel<<<(unsigned)cblocks, 256, 0, stream>>>(p.colp, cols, p.bins, last_bin_nnz);
    if ((e = cudaGetLastError()) != cudaSuccess) return (int)e;
    std::vector<unsigned> bins(HOT_BINS);
    unsigned long long last = 0;
    if ((e = cudaMemcpyAsync(bins.data(), p.bins, HOT_BINS * sizeof(unsigned), cudaMemcpyDeviceToHost, stream)) != cudaSuccess ||
        (e = cudaMemcpyAsync(&last, last_bin_nnz, sizeof last, cudaMemcpyDeviceToHost, stream)) != cudaSuccess ||
        (e = cudaStreamSynchronize(stream)) != cudaSuccess)
        return (int)e;
    int tau = 0;
    const int nhot = flat_hot_choose(bins.data(), last, nnz, HOT_BYTES / (dtype == 1 ? 8 : 4), &tau);
    if (nhot == 0) return 0;
    const int64_t nb = (cols + SCAN_ITEMS - 1) / SCAN_ITEMS;      // the hot list, ascending: a scan over the columns
    HotFlag v{p.colp, tau};
    scan_block_sums_kernel<<<(unsigned)nb, 256, 0, stream>>>(v, cols, p.scratch);
    scan_of_block_sums_kernel<<<1, 1024, 0, stream>>>(p.scratch, nb, p.ctl + 8);
    scan_emit_kernel<<<(unsigned)nb, 256, 0, stream>>>(v, EmitHot{p.hot}, cols, p.scratch);
    int64_t kb = (npad + 255) / 256;
    if (kb > 132 * 32) kb = 132 * 32;
    flat_hot_colp_kernel<<<(unsigned)kb, 256, 0, stream>>>(col, base, nnz, npad, p.hot, nhot, tau, p.colp, p.ctl);
    if ((e = cudaGetLastError()) != cudaSuccess) return (int)e;
    *hot_out = nhot;
    return 0;
}

void b200spmv_csr_flat_hot_offsets(int64_t rows, int64_t nnz, size_t* colp, size_t* hot) {
    FlatPlan p;
    flat_layout(rows, nnz, nullptr, &p);
    if (colp) *colp = (size_t)((char*)p.colp - (char*)nullptr);
    if (hot) *hot = (size_t)((char*)p.hot - (char*)nullptr);
}

void b200spmv_csr_flat_hot_params(int32_t* hot_bytes, int32_t* min_share_permille, int32_t* bins) {
    if (hot_bytes) *hot_bytes = HOT_BYTES;
    if (min_share_permille) *min_share_permille = HOT_MIN_PERMILLE;
    if (bins) *bins = HOT_BINS;
}

int b200spmv_csr_flat_mv(void* stream, int dtype, int64_t rows, int64_t cols, int64_t nnz, const void* row_offsets,
                         const void* col_ind, const void* values, int32_t base, const void* alpha, const void* beta,
                         int scalars_on_device, const void* x, void* y, void* workspace, int32_t hot) {
    if (rows < 0 || cols < 0 || nnz < 0 || !alpha || !beta) return -1;
    if (rows == 0) return 0;
    if (!y || !workspace || !row_offsets || (nnz > 0 && (!col_ind || !values || !x))) return -1;
    if (dtype == 0)
        return launch_flat<float>((cudaStream_t)stream, rows, nnz, row_offsets, col_ind, values, base, alpha, beta, scalars_on_device, x, y,
                                  workspace, hot);
    if (dtype == 1)
        return launch_flat<double>((cudaStream_t)stream, rows, nnz, row_offsets, col_ind, values, base, alpha, beta, scalars_on_device, x, y,
                                   workspace, hot);
    return -1;
}

}  // extern "C"
