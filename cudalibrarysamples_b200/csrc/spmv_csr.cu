// spmv_csr.cu -- CSR  y = alpha*A*x + beta*y  for H100 (sm_90a), fp32 / fp64, int32 indices.
//
// Replaces the closed cusparse::partition_kernel / csrmv_v3_kernel / spmv_fixup_kernel trio behind
// cusparseSpMV_preprocess / cusparseSpMV (reference call sites: cuSPARSE/spmv_csr/spmv_csr_example.c:104-112,
// cuSPARSE/cg/cg_example.c:156,220,294,415, cuSPARSE/bicgstab/bicgstab_example.c:190,262,315,358,504).
//
// Design (DESIGN.md section 3):
//   * analyze (csr_partition_kernel): merge-path style partition of the (rows + nnz) item list into tiles of
//     TILE_ITEMS items.  A tile boundary that falls inside a row shorter than LONG_ROW is rounded down to that
//     row's start, so ordinary rows never straddle tiles and need no carry / fix-up; only rows >= LONG_ROW are cut.
//     Their covering tiles store one partial sum each; the partial sums are added in fixed tile order
//     (bit-reproducible) by csr_fixup_kernel (one-CTA-per-tile kernels; launched with programmatic stream
//     serialization) or by the last CTA to finish (persistent kernels) -- nothing waits inside a tile.
//   * mv: four kernels over the same plan, picked at run time (launch_csr):
//       csr_tile_kernel    one CTA per tile, products staged in shared memory          (default for >= 12 nnz/row)
//       csr_pipe_kernel    persistent CTAs, next tile's stream prefetched in registers (default for short rows)
//       csr_ws_kernel      warp-specialised, TMA (cp.async.bulk + mbarrier) fed        (experimental)
//       csr_rowwise_kernel no shared memory, lane groups own rows                      (experimental)
//     Common to all: every warp-level load / gather covers 32 consecutive non-zeros (aligned 128 B / 256 B stream
//     segments through ld.global.nc.L1::no_allocate, fewest distinct lines per x gather), rows are reduced by
//     groups of g = 1..32 lanes (g picked per tile from its mean row length) with a warp-shuffle tree, y is
//     written once.  No tensor cores: 0.125-0.17 flop/B.
//   * What bounds it (profiles/): on scattered matrices not HBM but the SM's L1TEX pipe, which serves x gathers
//     (~1 distinct line per clock), shared-memory accesses and shuffles strictly in order.
#include "spmv_common.cuh"
#include "config.h"
#include "../../include/b200spmv.h"
#include <cstdlib>
#include <cstring>
#include <mutex>

namespace b200 {

// Tunables (overridable with -D for the parameter sweeps in scripts/sweep.py).  The defaults here and in the other kernel
// files were swept on an earlier GPU and carried over unchanged; they have not been re-swept on the H100.
#ifndef B200_CSR_TILE_ITEMS
#define B200_CSR_TILE_ITEMS 2048
#endif
#ifndef B200_CSR_LONG_ROW
#define B200_CSR_LONG_ROW 512
#endif
#ifndef B200_CSR_BLOCK
#define B200_CSR_BLOCK 256
#endif
#ifndef B200_CSR_BATCH
#define B200_CSR_BATCH 4
#endif
#ifndef B200_CSR_MIN_CTAS        // -D override for sweeps: resident CTAs per SM the register allocator must allow
#define B200_TILE_MIN_CTAS 5     // one-CTA-per-tile kernel: 48 registers
#define B200_PIPE_MIN_CTAS 3     // persistent pipelined kernel: 80 registers (next tile's stream lives in registers)
#define B200_RW_MIN_CTAS 4
#else
#define B200_TILE_MIN_CTAS B200_CSR_MIN_CTAS
#define B200_PIPE_MIN_CTAS B200_CSR_MIN_CTAS
#define B200_RW_MIN_CTAS B200_CSR_MIN_CTAS
#endif
#ifndef B200_CSR_KERNEL      // -D override for sweeps: -1 = runtime choice (default), 0 = one CTA per tile,
#define B200_CSR_KERNEL -1   //  1 = persistent software-pipelined CTAs, 2 = warp-specialised TMA-fed, 3 = row-wise
#endif
#ifndef B200_CSR_PIPE_STEPS
#define B200_CSR_PIPE_STEPS ((B200_CSR_TILE_ITEMS + B200_CSR_BLOCK - 1) / B200_CSR_BLOCK)
#endif
#ifndef B200_CSR_PIPE_OFFS
#define B200_CSR_PIPE_OFFS 4
#endif
#ifndef B200_CSR_RED_ROWS     // rows a lane group reduces concurrently in phase 2
#define B200_CSR_RED_ROWS 2
#endif
#ifndef B200_CSR_RED_BUTTERFLY
#define B200_CSR_RED_BUTTERFLY 1
#endif
#ifndef B200_CSR_RED_U        // predicated product loads per lane and row before the fall-back loop
#define B200_CSR_RED_U 2
#endif
#ifndef B200_CSR_SOFF16    // stage the tile's rowOff slice as 16-bit offsets (5 KB less shared memory per CTA)
#define B200_CSR_SOFF16 1
#endif
#ifndef B200_CSR_ABLATE   // profiling only: 1 = skip phase 2, 2 = no x gather, 3 = neither (stream only)
#define B200_CSR_ABLATE 0
#endif
constexpr int CSR_TILE_ITEMS = B200_CSR_TILE_ITEMS;  // merge items (row ends + non-zeros) per tile
constexpr int CSR_LONG_ROW   = B200_CSR_LONG_ROW;    // rows at least this long may be split between tiles
constexpr int CSR_BLOCK      = B200_CSR_BLOCK;       // threads per CTA
constexpr int CSR_SMEM_ELEMS = CSR_TILE_ITEMS + CSR_LONG_ROW;  // max non-zeros a tile can hold
#if B200_CSR_SOFF16
typedef short soff_t;      // tile-relative row starts lie in [-1 (clamped), CSR_SMEM_ELEMS + 31] -- fits 16 bits
static_assert(B200_CSR_TILE_ITEMS + B200_CSR_LONG_ROW + 32 < 32767, "tile too large for 16-bit staged offsets");
#else
typedef int soff_t;
#endif
__device__ __forceinline__ soff_t to_soff(int v) { return (soff_t)(v < -1 ? -1 : v); }
constexpr int CSR_BATCH      = B200_CSR_BATCH;  // load steps whose loads are all issued before the first use
// a tile's element range starts at a multiple of 32 (<= 31 masked lanes) and holds < CSR_SMEM_ELEMS non-zeros
constexpr int CSR_STEPS      = (CSR_SMEM_ELEMS + 31 + CSR_BLOCK - 1) / CSR_BLOCK;
constexpr int CSR_ITERS      = (CSR_STEPS + CSR_BATCH - 1) / CSR_BATCH * CSR_BATCH;

constexpr size_t PLAN_HEADER_BYTES = 256;

struct PlanView {
    int2*   tiles;      // [num_tiles+1] (row, nnz) start coordinate of each tile
    int*    ctl;        // [0] = arrivals of the current launch, [1] = number of split rows, [2] = number of partial sums (analyze)
    int4*   split;      // [num_tiles+1] split rows: (row, first covering tile b1, last covering tile b2, -)
    double* head_part;  // [num_tiles+1] partial sum of the split row a tile starts in
    double* tail_part;  // [num_tiles+1] partial sum of the split row a tile ends in
};

static inline int64_t csr_num_tiles(int64_t rows, int64_t nnz) {
    return (rows + nnz + CSR_TILE_ITEMS - 1) / CSR_TILE_ITEMS;
}

static inline size_t plan_layout(int64_t num_tiles, void* ws, PlanView* v) {
    size_t n = (size_t)num_tiles + 1;
    size_t o_tiles = PLAN_HEADER_BYTES;
    size_t o_ctl   = round_up_256(o_tiles + n * sizeof(int2));
    size_t o_split = round_up_256(o_ctl + 64);
    size_t o_head  = round_up_256(o_split + n * sizeof(int4));
    size_t o_tail  = round_up_256(o_head + n * sizeof(double));
    size_t total   = round_up_256(o_tail + n * sizeof(double));
    if (v) {
        char* b = (char*)ws;
        v->tiles = (int2*)(b + o_tiles);
        v->ctl = (int*)(b + o_ctl);
        v->split = (int4*)(b + o_split);
        v->head_part = (double*)(b + o_head);
        v->tail_part = (double*)(b + o_tail);
    }
    return total;
}

// ------------------------------------------------------------------------------------------------
// analyze: one thread per tile boundary.
//   boundary b sits on merge diagonal d = min(b*TILE, rows+nnz); r = the row the diagonal cuts
//   (largest r with r + off[r] <= d).  Rows shorter than LONG_ROW are never cut: the boundary moves to
//   the row start (r, off[r]); long rows are cut exactly at the diagonal (r, off[r] + e).
// ------------------------------------------------------------------------------------------------
__global__ void csr_partition_kernel(const int* __restrict__ off, int base, int64_t rows, int64_t nnz,
                                     int64_t num_tiles, PlanView plan) {
    int64_t b = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (b > num_tiles) return;
    int64_t d = b * CSR_TILE_ITEMS;
    if (d > rows + nnz) d = rows + nnz;
    int64_t lo = 0, hi = rows;
    while (lo < hi) {
        int64_t mid = (lo + hi + 1) >> 1;
        if (mid + (int64_t)(off[mid] - base) <= d) lo = mid; else hi = mid - 1;
    }
    int64_t r = lo, n = off[r] - base;
    if (r < rows) {
        int64_t len = (int64_t)(off[r + 1] - base) - n;
        int64_t e = d - (r + n);
        if (len >= CSR_LONG_ROW && e > 0) {
            // Row r is cut here.  It is covered by tiles b1 = g(r)/TILE (holding its start as a "tail") through
            // b2 = (g(r)+len)/TILE (the others hold "heads"); the boundary that makes the FIRST cut registers the row
            // in the split list that the fix-up pass walks.
            const int64_t g0 = r + n, b1 = g0 / CSR_TILE_ITEMS, b2 = (g0 + len) / CSR_TILE_ITEMS;
            if (b == b1 + 1) {
                const int slot = atomicAdd(plan.ctl + 1, 1);
                plan.split[slot] = make_int4((int)r, (int)b1, (int)b2, 0);
                atomicAdd(plan.ctl + 2, (int)(b2 - b1 + 1));   // partial sums the covering tiles will deposit
            }
            n += e;
        }
    }
    plan.tiles[b] = make_int2((int)r, (int)n);
    plan.head_part[b] = 0.0;
    plan.tail_part[b] = 0.0;
}

#ifdef B200_CSR_TRACE   // debugging builds only: per-tile clock64 stamps {start, after phase 1, end, smid}
#define TRACE_STAMP(a, b, slot) do { if ((a).trace && threadIdx.x == 0) (a).trace[(size_t)(b) * 4 + (slot)] = clock64(); } while (0)
#define TRACE_SMID(a, b) do { if ((a).trace && threadIdx.x == 0) { unsigned s_; asm volatile("mov.u32 %0, %%smid;" : "=r"(s_)); (a).trace[(size_t)(b) * 4 + 3] = s_; } } while (0)
static long long* g_trace_ptr = nullptr;
extern "C" void b200spmv_debug_set_trace(void* p) { g_trace_ptr = (long long*)p; }
#else
#define TRACE_STAMP(a, b, slot) do { } while (0)
#define TRACE_SMID(a, b) do { } while (0)
#endif

template <typename T>
struct CsrArgs {
    const int* off;
    const int* col;
    const T*   val;
    const T*   x;
    T*         y;
    int        base;
    int        rows;
    int        nnz;
    Scalars<T> s;
    PlanView   plan;
    long long* trace;
    unsigned   tile_stride;   // one-CTA-per-tile kernels visit tile (blockIdx * tile_stride) % num_tiles (1 = in order)
    unsigned   num_tiles;
    int        seg_dense;     // csr_seg_kernel: tiles with >= seg_dense non-zeros per row end take the register path
    int        pdl;           // 1: the fix-up kernel is launched with programmatic stream serialization (opt-in)
};

// The phase-2 code runs either on a whole CTA (tile / pipe kernels: __syncthreads) or on the "reduce" warps of a
// warp-specialised CTA (named barrier BAR_ID over BLOCK threads); `tid` is the thread's index inside that group.
template <int BLOCK, int BAR_ID>
__device__ __forceinline__ void group_sync() {
    if (BAR_ID == 0) __syncthreads();
    else asm volatile("bar.sync %0, %1;" ::"n"(BAR_ID), "n"(BLOCK) : "memory");
}

// Sum sP[lo, hi) with the whole group, fixed order (bit-reproducible). Result valid on group thread 0.
template <typename T, int BLOCK, int BAR_ID>
__device__ __forceinline__ T block_sum_range(const T* sP, int lo, int hi, T* sRed, int tid) {
    T s = T(0);
    for (int k = lo + tid; k < hi; k += BLOCK) s += sP[k];
    s = warp_sum(s);
    group_sync<BLOCK, BAR_ID>();  // sRed reuse
    if ((tid & 31) == 0) sRed[tid >> 5] = s;
    group_sync<BLOCK, BAR_ID>();
    T tot = T(0);
    if (tid == 0) {
#pragma unroll
        for (int w = 0; w < BLOCK / 32; w++) tot += sRed[w];
    }
    return tot;
}

// Rows [r_first, r_first + nrows) are complete inside the tile; the products of row r live at
// sP[sOff[r - rs] .. sOff[r - rs + 1]) (sOff = the tile's slice of rowOff, staged in phase 1, rebased to the tile).
//
// Every shared-memory access and every shuffle of this phase queues in the SM's single L1TEX FIFO behind the x
// gathers of the other resident warps, so what matters is the NUMBER OF DEPENDENT STEPS, not the instruction count:
// a group of G lanes therefore works on ROWS rows at once -- all row bounds first, then all products (U predicated
// loads per lane and row, enough for rows up to U*G long), then ROWS interleaved shuffle trees.
constexpr int RED_ROWS = B200_CSR_RED_ROWS;
constexpr int RED_ROWS4 = B200_CSR_RED_BUTTERFLY ? 4 : B200_CSR_RED_ROWS;   // groups of >= 4 lanes: 4 rows + transposed butterfly
constexpr int RED_U    = B200_CSR_RED_U;

template <typename T, typename OT, int G, int ROWS, int U, int BLOCK>
__device__ __forceinline__ void reduce_rows(const CsrArgs<T>& a, const T* sP, const OT* sOff, int shift, int rs,
                                            int r_first, int nrows, T alpha, T beta, int tid) {
    constexpr int GROUPS = BLOCK / G;
    const int gid = tid / G, gl = tid % G;
    const OT* so = sOff + (r_first - rs);
    for (int r0 = 0; r0 < nrows; r0 += GROUPS * ROWS) {
        int k0[ROWS], e[ROWS];
#pragma unroll
        for (int i = 0; i < ROWS; i++) {
            const int ri = r0 + i * GROUPS + gid;
            const bool active = ri < nrows;
            k0[i] = (active ? (int)so[ri] - shift : 0) + gl;
            e[i]  = active ? (int)so[ri + 1] - shift : 0;
        }
        T p[ROWS][U];
#pragma unroll
        for (int i = 0; i < ROWS; i++)
#pragma unroll
            for (int u = 0; u < U; u++) {
                const int k = k0[i] + u * G;
                p[i][u] = k < e[i] ? sP[k] : T(0);
            }
        T sum[ROWS];
#pragma unroll
        for (int i = 0; i < ROWS; i++) {
            sum[i] = p[i][0];
#pragma unroll
            for (int u = 1; u < U; u++) sum[i] += p[i][u];
        }
#pragma unroll
        for (int i = 0; i < ROWS; i++) {                        // rows longer than U*G: batches of U loads in flight
            for (int kb = k0[i] + U * G; kb < e[i]; kb += U * G) {
                T q[U];
#pragma unroll
                for (int u = 0; u < U; u++) q[u] = kb + u * G < e[i] ? sP[kb + u * G] : T(0);
#pragma unroll
                for (int u = 0; u < U; u++) sum[i] += q[u];
            }
        }
        if (ROWS == 4 && G >= 4) {
            // Transposed butterfly: 4 row sums over G lanes in 2 + 1 + log2(G/4) exchanges instead of 4*log2(G)
            // (shuffles queue in the same L1TEX pipe as the gathers).  After the first two exchanges every lane of
            // quarter q = 2*hi + mid of the group carries one partial of row slot q.
            const bool hi = (gl & (G / 2)) != 0, mid = (gl & (G / 4)) != 0;
            const T s0 = hi ? sum[0] : sum[2], s1 = hi ? sum[1] : sum[3];
            T k0v = (hi ? sum[2] : sum[0]) + __shfl_xor_sync(0xffffffffu, s0, G / 2);
            T k1v = (hi ? sum[3] : sum[1]) + __shfl_xor_sync(0xffffffffu, s1, G / 2);
            T kv  = (mid ? k1v : k0v) + __shfl_xor_sync(0xffffffffu, mid ? k0v : k1v, G / 4);
#pragma unroll
            for (int o = G / 8; o > 0; o >>= 1) kv += __shfl_xor_sync(0xffffffffu, kv, o);
            if ((gl & (G / 4 - 1)) == 0) {
                const int slot = (hi ? 2 : 0) + (mid ? 1 : 0);
                const int ri = r0 + slot * GROUPS + gid;
                if (ri < nrows) {
                    T* yp = a.y + r_first + ri;
                    *yp = axpby(alpha, kv, beta, yp);
                }
            }
        } else {
#pragma unroll
            for (int o = G / 2; o > 0; o >>= 1)
#pragma unroll
                for (int i = 0; i < ROWS; i++) sum[i] += __shfl_down_sync(0xffffffffu, sum[i], o, G);
            if (gl == 0) {
#pragma unroll
                for (int i = 0; i < ROWS; i++) {
                    const int ri = r0 + i * GROUPS + gid;
                    if (ri < nrows) {
                        T* yp = a.y + r_first + ri;
                        *yp = axpby(alpha, sum[i], beta, yp);
                    }
                }
            }
        }
    }
}

// y[R] = alpha * (tail_part[b1] + head_part[b1+1] + ... + head_part[b2]) + beta * y[R] for every split row, by one
// CTA (or, from the fix-up kernel, by the whole grid), in fixed tile order (bit-reproducible).  Four rows per thread are in flight at a time: the loads of one row are
// a dependent chain of L2 round trips, and a 10 M-row R-MAT has ~10^5 partial sums to add.
template <typename T>
__device__ __forceinline__ void sum_split_rows(const CsrArgs<T>& a, T alpha, T beta, bool whole_grid = false) {
    constexpr int RU = 4;
    const int nsplit = __ldcg(a.plan.ctl + 1);
    const int nthr = (int)blockDim.x * (whole_grid ? (int)gridDim.x : 1);
    for (int i0 = (int)threadIdx.x + (whole_grid ? (int)(blockIdx.x * blockDim.x) : 0); i0 < nsplit; i0 += RU * nthr) {
        int4   sr[RU];
        double sum[RU], h1[RU];
#pragma unroll
        for (int j = 0; j < RU; j++) {
            const int i = i0 + j * nthr;
            sr[j] = i < nsplit ? a.plan.split[i] : make_int4(-1, 0, -1, 0);
        }
#pragma unroll
        for (int j = 0; j < RU; j++) {
            const bool live = sr[j].x >= 0;
            sum[j] = live ? __ldcg(a.plan.tail_part + sr[j].y) : 0.0;
            h1[j]  = (live && sr[j].z > sr[j].y) ? __ldcg(a.plan.head_part + sr[j].y + 1) : 0.0;
        }
#pragma unroll
        for (int j = 0; j < RU; j++) {
            sum[j] += h1[j];
            for (int b = sr[j].y + 2; b <= sr[j].z; b++) sum[j] += __ldcg(a.plan.head_part + b);   // rows cut more than once
            if (sr[j].x >= 0) {
                T* yp = a.y + sr[j].x;
                *yp = axpby(alpha, (T)sum[j], beta, yp);
            }
        }
    }
}

// Split rows (>= LONG_ROW non-zeros, cut by a tile boundary): every covering tile only STORES its partial sum
// (head_part[b] / tail_part[b], fire-and-forget, nothing waits).  When a CTA has finished all its tiles it bumps
// ctl[0]; the CTA that arrives last walks the split list built by analyze and writes
//     y[R] = alpha * (tail_part[b1] + head_part[b1+1] + ... + head_part[b2]) + beta * y[R]
// in fixed tile order -> bit-reproducible, single launch, no spin-waits, counter left at 0 for the next launch.
template <typename T>
__device__ __forceinline__ void split_rows_fixup(const CsrArgs<T>& a, T alpha, T beta) {
    __shared__ int s_last;
    __threadfence();                       // this CTA's partial sums are visible device-wide
    __syncthreads();
    if (threadIdx.x == 0) {
        const int old = atomicAdd(a.plan.ctl, 1);
        s_last = old == (int)gridDim.x - 1;
    }
    __syncthreads();
    if (!s_last) return;
    __threadfence();
    sum_split_rows<T>(a, alpha, beta);
    if (threadIdx.x == 0) a.plan.ctl[0] = 0;
}

// ---------------- phase 2: per-row reduction out of shared memory ----------------------------------
// sP[0 .. ne-ns) holds the tile's products, sOff[i] - shift = rowOff[rs+i] - base - ns for i = 0 .. re-rs (the
// tile / pipe kernels stage rebased offsets, shift = 0; the TMA-fed kernel stages the raw slice, shift = base + ns).
template <typename T, typename OT, int BLOCK, int BAR_ID>
__device__ __forceinline__ int tile_phase2(const CsrArgs<T>& a, int b, int rs, int ns, int re, int ne, const T* sP,
                                           const OT* sOff, int shift, T* sRed, T alpha, T beta, int tid) {
    if (B200_CSR_ABLATE & 1) { if (sP[tid] == T(1.2345)) a.y[0] = sP[0]; return 0; }
    const int cnt = ne - ns;
    bool head = false;
    int  head_end = 0;  // products [0, head_end) belong to the split row rs
    if (rs < a.rows && (int)sOff[0] - shift < 0) {       // the tile starts inside row rs
        head = true;
        const int o1 = re > rs ? (int)sOff[1] - shift : cnt;  // re == rs: the whole tile lies inside row rs
        head_end = o1 < cnt ? o1 : cnt;
    }
    const int r_first = rs + (head ? 1 : 0);
    const int nrows   = re - r_first;  // complete rows (may be <= 0)
    int  tail_beg = cnt;               // products [tail_beg, cnt) belong to the split row re
    bool tail = false;
    if (re < a.rows && re >= r_first) {
        const int o0 = (int)sOff[re - rs] - shift;
        if (cnt > o0) { tail = true; tail_beg = o0; }
    }

    if (nrows > 0) {
        const int body = tail_beg - head_end;
        const int avg2 = body / (2 * nrows);  // half the mean row length
        if      (avg2 <= 1)  reduce_rows<T, OT, 1, RED_ROWS, RED_U, BLOCK>(a, sP, sOff, shift, rs, r_first, nrows, alpha, beta, tid);
        else if (avg2 <= 2)  reduce_rows<T, OT, 2, RED_ROWS, RED_U, BLOCK>(a, sP, sOff, shift, rs, r_first, nrows, alpha, beta, tid);
        else if (avg2 <= 4)  reduce_rows<T, OT, 4, RED_ROWS4, RED_U, BLOCK>(a, sP, sOff, shift, rs, r_first, nrows, alpha, beta, tid);
        else if (avg2 <= 8)  reduce_rows<T, OT, 8, RED_ROWS4, RED_U, BLOCK>(a, sP, sOff, shift, rs, r_first, nrows, alpha, beta, tid);
        else if (avg2 <= 16) reduce_rows<T, OT, 16, RED_ROWS4, RED_U, BLOCK>(a, sP, sOff, shift, rs, r_first, nrows, alpha, beta, tid);
        else                 reduce_rows<T, OT, 32, 2, 8, BLOCK>(a, sP, sOff, shift, rs, r_first, nrows, alpha, beta, tid);  // long rows: 256 elements per batch
    }

    if (head) {  // group-uniform
        const T hs = block_sum_range<T, BLOCK, BAR_ID>(sP, 0, head_end, sRed, tid);
        if (tid == 0) a.plan.head_part[b] = (double)hs;
    }
    if (tail) {  // group-uniform
        const T ts = block_sum_range<T, BLOCK, BAR_ID>(sP, tail_beg, cnt, sRed, tid);
        if (tid == 0) a.plan.tail_part[b] = (double)ts;
    }
    return (head ? 1 : 0) + (tail ? 1 : 0);   // partial sums this tile deposited (group-uniform)
}


// One CTA per tile; products of the whole tile staged in shared memory, rows reduced by lane groups (tile_phase2).
template <typename T>
__global__ void __launch_bounds__(CSR_BLOCK, B200_TILE_MIN_CTAS) csr_tile_kernel(const CsrArgs<T> a) {
    __shared__ T   sP[CSR_SMEM_ELEMS];
    __shared__ soff_t sOff[CSR_SMEM_ELEMS + 1];   // rowOff[rs .. re] - base - ns: a tile spans < CSR_SMEM_ELEMS rows
    __shared__ T   sRed[CSR_BLOCK / 32];

    // Tiles are visited in a scattered order: neighbouring tiles of a skewed matrix look alike (R-MAT: long rows first,
    // thousands of near-empty rows later), and the SM overlaps a gather-heavy tile best with a row-heavy one.
    const int  b  = (int)(((unsigned long long)blockIdx.x * a.tile_stride) % a.num_tiles);
    const int2 st = a.plan.tiles[b], en = a.plan.tiles[b + 1];
    const int  rs = st.x, ns = st.y, re = en.x, ne = en.y;
    const T alpha = a.s.a(), beta = a.s.b();
    TRACE_STAMP(a, b, 0); TRACE_SMID(a, b);
    if (a.pdl) cudaTriggerProgrammaticLaunchCompletion();   // lets csr_fixup_kernel get resident early (it still waits for our completion)

    // ---------------- phase 1: stream val/col, gather x, park products in shared memory -------------
    // Lane l of a warp handles element (step*BLOCK + warp*32 + l): every load/gather instruction covers 32
    // CONSECUTIVE non-zeros.  The streaming loads are then perfectly coalesced (the tile's first element is
    // rounded down to a multiple of 32 so each warp-level load is one aligned 128 B / 256 B segment), the
    // gathers of x see the sorted neighbouring columns of a row in one instruction (fewest L1TEX wavefronts:
    // the gather rate of the SM, ~1 distinct 128 B line per clock, is what bounds this kernel on scattered
    // matrices), and the shared-memory stores are bank-conflict free.
    {
        // the tile's slice of rowOff goes to shared memory first: its latency overlaps the val/col stream, and
        // phase 2 then never waits on global memory
        const int noff = (re < a.rows ? re : a.rows) - rs + 1;
        for (int i = (int)threadIdx.x; i < noff; i += CSR_BLOCK) sOff[i] = to_soff(__ldg(a.off + rs + i) - a.base - ns);
        const int al   = ns & ~31;
        const int lead = ns - al;                 // masked lanes in front of the tile
        const int span = ne - al;                 // elements [lead, span) are live
        const int* colp = a.col + al;
        const T*   valp = a.val + al;
#pragma unroll
        for (int batch = 0; batch < CSR_ITERS; batch += CSR_BATCH) {
            if (batch * CSR_BLOCK < span) {       // block-uniform
                int c[CSR_BATCH];
                T   v[CSR_BATCH], xv[CSR_BATCH];
#pragma unroll
                for (int k = 0; k < CSR_BATCH; k++) {
                    const int e = (batch + k) * CSR_BLOCK + (int)threadIdx.x;
                    const bool live = e >= lead && e < span;
                    c[k] = live ? ldg_stream(colp + e) : a.base;
                    v[k] = live ? ldg_stream(valp + e) : T(0);
                }
#pragma unroll
                for (int k = 0; k < CSR_BATCH; k++) {
                    const int e = (batch + k) * CSR_BLOCK + (int)threadIdx.x;
                    const bool live = e >= lead && e < span;
                    xv[k] = (live && !(B200_CSR_ABLATE & 2)) ? __ldg(a.x + (c[k] - a.base)) : T(c[k]);
                }
#pragma unroll
                for (int k = 0; k < CSR_BATCH; k++) {
                    const int e = (batch + k) * CSR_BLOCK + (int)threadIdx.x;
                    if (e >= lead && e < span) sP[e - lead] = v[k] * xv[k];
                }
            }
        }
    }
    __syncthreads();
    TRACE_STAMP(a, b, 1);

    tile_phase2<T, soff_t, CSR_BLOCK, 0>(a, b, rs, ns, re, ne, sP, sOff, 0, sRed, alpha, beta, (int)threadIdx.x);
    TRACE_STAMP(a, b, 2);
}

// ================================================================================================
// csr_seg_kernel ("seg"): one CTA per tile, but the products of ROW-SPARSE tiles never touch shared memory.
//
// Why (profiles/ncu_r1_summary_table.md, ncu of csr_tile_kernel on R-MAT 1M): the kernel is bound by the SM's L1TEX
// data pipe (19.4 M wavefronts per launch: 12.4 M global, 1.1 M STS, 2.3 M LDS, 3.6 M SHFL), and a third of that is the
// row reduction: every product makes a round trip through shared memory and every row -- whatever its length -- pays
// a full shuffle tree of its tile's group size.  On skewed matrices 81 % of the non-zeros sit in rows >= 32 long.
//
// Here every warp owns a CONTIGUOUS chunk of the tile (still 32 consecutive non-zeros per load / gather instruction)
// and walks it step by step with a per-lane accumulator:
//   * a 32-element step in which no row ends costs nothing: acc += product;
//   * a step in which rows end: the lanes hold a window of the next 32 row ends (from the staged rowOff slice); one
//     ballot finds the k rows ending in this step, one REDUX.OR builds the mask of their end lanes, ONE butterfly
//     gives the first row's total (accumulator + head of the step), a segmented shuffle scan -- only as many levels as
//     the longest remaining segment needs -- gives the others, and lane j fetches the total of row cur + j with one
//     shuffle and writes y[row cur + j] (coalesced; empty rows fall out as zero sums).
// Rows that cross chunk borders are stitched from <= 2 partials per warp by one thread after a barrier; rows that cross
// TILE borders (>= LONG_ROW) deposit head/tail partials for csr_fixup_kernel exactly like the other kernels.
// Modelled on the R-MAT 1M structure (scripts/model_seg_cost.py): 2.8 M shuffle wavefronts instead of 7.0 M
// shared + shuffle wavefronts.  Tiles with many short rows (more than one row per SEG_DENSE non-zeros) keep the
// staged-product path of csr_tile_kernel: there nearly every step ends several rows and the scan would cost more.
// ================================================================================================
#ifndef B200_SEG_BATCH
#define B200_SEG_BATCH 4
#endif
#ifndef B200_SEG_MIN_CTAS
#define B200_SEG_MIN_CTAS B200_TILE_MIN_CTAS
#endif
#ifndef B200_SEG_STAGED      // 0 (sweeps): no staged-product fallback, every tile takes the register path and the CTA needs
#define B200_SEG_STAGED 1    //   5 KB instead of 26 KB of shared memory (more of the unified L1 left for x)
#endif
constexpr int SEG_WARPS  = CSR_BLOCK / 32;
constexpr int SEG_WSTEPS = ((CSR_SMEM_ELEMS + 31 + 31) / 32 + SEG_WARPS - 1) / SEG_WARPS;   // 32-element steps per warp, worst case
constexpr int SEG_BATCH  = B200_SEG_BATCH;
constexpr int SEG_BIG    = 32767;                 // "this row never ends here": sentinel behind the staged row starts

// Number of j in [0, nr) with S[j + 1] <= lo  (S = staged row starts, non-decreasing), by the whole warp: two levels of
// a 32-ary search instead of log2(nr) dependent probes.
__device__ __forceinline__ int warp_count_ended(const soff_t* S, int nr, int lo, int lane) {
    if (nr <= 0) return 0;
    const int stride = (nr + 31) >> 5;
    const int blk_lo = lane * stride;
    const int blk_hi = min(blk_lo + stride, nr);                         // block [blk_lo, blk_hi)
    const bool full = blk_lo < nr && (int)S[blk_hi] <= lo;               // the block's last row has ended
    const int nb = __popc(__ballot_sync(0xffffffffu, full));
    int cnt = nb * stride;
    if (cnt >= nr) return nr;
    const int hi = min(cnt + stride, nr);
    int extra = 0;
    for (int j0 = cnt; j0 < hi; j0 += 32) {                              // warp-uniform trip count (<= 3)
        const int j = j0 + lane;
        extra += __popc(__ballot_sync(0xffffffffu, j < hi && (int)S[j + 1] <= lo));
    }
    return cnt + extra;
}

template <typename T>
__global__ void __launch_bounds__(CSR_BLOCK, B200_SEG_MIN_CTAS) csr_seg_kernel(const CsrArgs<T> a) {
#if B200_SEG_STAGED
    __shared__ T      sP[CSR_SMEM_ELEMS];
    __shared__ T      sRed[SEG_WARPS];
#endif
    __shared__ soff_t sOff[CSR_SMEM_ELEMS + 1 + 34];      // row starts of the tile + 33 sentinels for the lane window
    __shared__ T      sFirst[SEG_WARPS], sOpen[SEG_WARPS];
    __shared__ int    sFirstRow[SEG_WARPS];               // >= 0: the chunk ended at least one row; its first one is this row

    const int  b  = (int)(((unsigned long long)blockIdx.x * a.tile_stride) % a.num_tiles);
    const int2 st = a.plan.tiles[b], en = a.plan.tiles[b + 1];
    const int  rs = st.x, ns = st.y, re = en.x, ne = en.y;
    const T alpha = a.s.a(), beta = a.s.b();
    if (a.pdl) cudaTriggerProgrammaticLaunchCompletion();
    const int tid = (int)threadIdx.x, warp = tid >> 5, lane = tid & 31;

    const int nr  = re - rs;                  // rows [rs, re) END in this tile (merge path: a row's end item follows its non-zeros)
    const int cnt = ne - ns;
    const int noff = nr + 1;                  // S(0 .. nr); re <= rows, so rowOff[re] exists
    for (int i = tid; i < noff; i += CSR_BLOCK) sOff[i] = to_soff(__ldg(a.off + rs + i) - a.base - ns);
    if (tid < 34) sOff[noff + tid] = (soff_t)SEG_BIG;

    const int al = ns & ~31, lead = ns - al, span = ne - al;
    const int* colp = a.col + al;
    const T*   valp = a.val + al;
#if B200_SEG_STAGED
    const bool sparse = cnt >= a.seg_dense * (nr > 0 ? nr : 1);   // block-uniform, from the tile descriptor alone

    if (!sparse) {
        // ---------------- many short rows: products staged in shared memory, as in csr_tile_kernel ----------------
#pragma unroll
        for (int batch = 0; batch < CSR_ITERS; batch += CSR_BATCH) {
            if (batch * CSR_BLOCK < span) {
                int c[CSR_BATCH];
                T   v[CSR_BATCH], xv[CSR_BATCH];
#pragma unroll
                for (int k = 0; k < CSR_BATCH; k++) {
                    const int e = (batch + k) * CSR_BLOCK + tid;
                    const bool live = e >= lead && e < span;
                    c[k] = live ? ldg_stream(colp + e) : a.base;
                    v[k] = live ? ldg_stream(valp + e) : T(0);
                }
#pragma unroll
                for (int k = 0; k < CSR_BATCH; k++) {
                    const int e = (batch + k) * CSR_BLOCK + tid;
                    xv[k] = (e >= lead && e < span) ? __ldg(a.x + (c[k] - a.base)) : T(0);
                }
#pragma unroll
                for (int k = 0; k < CSR_BATCH; k++) {
                    const int e = (batch + k) * CSR_BLOCK + tid;
                    if (e >= lead && e < span) sP[e - lead] = v[k] * xv[k];
                }
            }
        }
        __syncthreads();
        tile_phase2<T, soff_t, CSR_BLOCK, 0>(a, b, rs, ns, re, ne, sP, sOff, 0, sRed, alpha, beta, tid);
        return;
    }
#else
    if (cnt == 0) {                           // only empty rows end here: y = beta * y (a split row that ends here deposits 0)
        __syncthreads();
        for (int j = tid; j < nr; j += CSR_BLOCK) {
            if (j == 0 && (int)sOff[0] < 0) a.plan.head_part[b] = 0.0;
            else { T* yp = a.y + rs + j; *yp = axpby(alpha, T(0), beta, yp); }
        }
        return;
    }
#endif

    // ---------------- row-sparse tile: warp w owns steps [s0, s0 + steps_w) of the tile ----------------
    const int steps_total = (span + 31) >> 5;
    const int steps_w = (steps_total + SEG_WARPS - 1) / SEG_WARPS;       // block-uniform, 1 .. SEG_WSTEPS
    const int s0 = warp * steps_w;
    const int cs = max(s0 * 32 - lead, 0);                               // chunk = tile-relative positions [cs, ce)
    const int ce = min((s0 + steps_w) * 32 - lead, cnt);
    const bool active = cs < ce;

    // walk state; cur / frow / acc_live are warp-uniform, ws / we / acc per lane
    int  cur = 0, frow = -1;
    int  ws = SEG_BIG, we = SEG_BIG;          // lane j: start / end (exclusive) of row cur + j, tile-relative
    T    acc = T(0), first = T(0);
    bool acc_live = false;                    // some lane of acc may be non-zero

    int c[SEG_BATCH];
    T   v[SEG_BATCH];
#pragma unroll
    for (int k = 0; k < SEG_BATCH; k++) {     // first batch of the stream in flight before anything else
        const int e = (s0 + k) * 32 + lane;
        const bool live = k < steps_w && e >= lead && e < span;
        c[k] = live ? ldg_stream(colp + e) : a.base;
        v[k] = live ? ldg_stream(valp + e) : T(0);
    }

    // Run-time loops on purpose (no unrolling over the steps): fully unrolled, the flush code below was instantiated 12
    // times and instruction-cache misses became the kernel's top stall reason.  Only the short load / gather loops over a
    // batch are unrolled.
#pragma unroll 1
    for (int kb = 0; kb < steps_w; kb += SEG_BATCH) {                    // block-uniform trip count
        T p[SEG_BATCH];
#pragma unroll
        for (int k = 0; k < SEG_BATCH; k++) {
            const int e = (s0 + kb + k) * 32 + lane;
            const bool live = kb + k < steps_w && e >= lead && e < span;
            p[k] = live ? v[k] * __ldg(a.x + (c[k] - a.base)) : T(0);
        }
        if (kb + SEG_BATCH < steps_w) {                                  // next batch of the stream (block-uniform)
#pragma unroll
            for (int k = 0; k < SEG_BATCH; k++) {
                const int e = (s0 + kb + SEG_BATCH + k) * 32 + lane;
                const bool live = kb + SEG_BATCH + k < steps_w && e >= lead && e < span;
                c[k] = live ? ldg_stream(colp + e) : a.base;
                v[k] = live ? ldg_stream(valp + e) : T(0);
            }
        }
        if (kb == 0) {
            __syncthreads();                                             // sOff is staged; the loads above are in flight
            if (active) {
                // rows whose end lies at or before the chunk start were finished by earlier warps (warp 0: none)
                cur = warp == 0 ? 0 : warp_count_ended(sOff, nr, cs, lane);
                ws = (int)sOff[cur + lane];
                we = (int)sOff[cur + lane + 1];
            }
        }
        if (!active) continue;
#pragma unroll 1
        for (int k = 0; k < SEG_BATCH; k++) {
            const int sb = (s0 + kb + k) * 32 - lead;                    // tile-relative position of lane 0
            if (kb + k >= steps_w || sb >= ce) break;                    // warp-uniform (the last warp's chunk may end early)
            const int step_end = min(sb + 32, ce);
            T pend = p[0];                                               // p[k] with a run-time k: a select chain, not local memory
#pragma unroll
            for (int j = 1; j < SEG_BATCH; j++) pend = k == j ? p[j] : pend;
#pragma unroll 1
            for (;;) {
                const int kk = __popc(__ballot_sync(0xffffffffu, we <= step_end));   // rows ending in this step
                if (kk == 0) break;
                const bool has = lane < kk && we > max(ws, cs);          // row cur + lane has elements in this chunk
                const unsigned m = __reduce_or_sync(0xffffffffu, has ? 1u << (we - 1 - sb) : 0u);
                T res = T(0);
                if (m != 0u) {
                    const int e1 = __ffs(m) - 1, ek = 31 - __clz(m);
                    const T t1 = warp_allsum(acc + (lane <= e1 ? pend : T(0)));
                    T q = (lane > e1 && lane <= ek) ? pend : T(0);
                    if (m & (m - 1u)) {                                  // more rows end: segmented inclusive scan
                        const unsigned below = m & ((1u << lane) - 1u);
                        const int dist = (lane > e1 && lane <= ek) ? lane - (32 - __clz(below)) : 0;   // lanes before me in my segment
#pragma unroll 1
                        for (int d = 1; d < 32; d <<= 1) {
                            if (__ballot_sync(0xffffffffu, dist >= d) == 0u) break;          // no segment that long
                            const T t = __shfl_up_sync(0xffffffffu, q, d);
                            if (dist >= d) q += t;
                        }
                    }
                    res = lane == e1 ? t1 : q;
                    acc = T(0);
                    acc_live = false;
                    pend = lane > ek ? pend : T(0);
                }
                T val = __shfl_sync(0xffffffffu, res, has ? we - 1 - sb : 0);
                val = has ? val : T(0);
                if (frow < 0) {                                          // the chunk's first row end goes to the stitcher
                    first = val;                                         // lane 0 keeps it (only lane 0 stores it)
                    frow = cur;
                    if (lane > 0 && lane < kk) {
                        T* yp = a.y + rs + cur + lane;
                        *yp = axpby(alpha, val, beta, yp);
                    }
                } else if (lane < kk) {
                    T* yp = a.y + rs + cur + lane;
                    *yp = axpby(alpha, val, beta, yp);
                }
                cur += kk;
                ws = (int)sOff[cur + lane];
                we = (int)sOff[cur + lane + 1];
                if (kk < 32) break;
            }
            acc += pend;
            acc_live = acc_live || __ballot_sync(0xffffffffu, pend != T(0)) != 0u;
        }
    }
    {
        const T open = acc_live ? warp_allsum(acc) : T(0);               // the row in progress continues past this chunk
        if (lane == 0) {
            if (frow >= 0) { sFirst[warp] = first; sOpen[warp] = open; }
            else           { sFirst[warp] = open;  sOpen[warp] = T(0); }  // no row ended: the whole chunk is one partial
            sFirstRow[warp] = frow;
        }
    }
    __syncthreads();

    if (tid == 0) {
        const bool head = (int)sOff[0] < 0;                              // the tile starts inside row rs (split row)
        T    running = T(0);
        bool any_end = false;
#pragma unroll
        for (int w = 0; w < SEG_WARPS; w++) {
            const int fr = sFirstRow[w];
            if (fr >= 0) {
                const T tot = running + sFirst[w];
                if (fr == 0 && head) a.plan.head_part[b] = (double)tot;
                else { T* yp = a.y + rs + fr; *yp = axpby(alpha, tot, beta, yp); }
                running = sOpen[w];
                any_end = true;
            } else {
                running += sFirst[w];
            }
        }
        if (head && !any_end) a.plan.head_part[b] = (double)running;    // the whole tile lies inside row rs
        else if (re < a.rows && cnt > (int)sOff[nr]) a.plan.tail_part[b] = (double)running;   // the tile ends inside row re
    }
}

// One-CTA-per-tile launches leave the split rows to this small second launch.  (Measured alternatives: an arrival
// counter bumped by every CTA, or only by the CTAs that deposited partial sums, is slower on R-MAT because a whole
// CTA waits for one atomic round trip; the extra launch is cheaper.)
template <typename T>
__global__ void __launch_bounds__(256) csr_fixup_kernel(const CsrArgs<T> a) {
    // When launched with programmatic stream serialization (opt-in) these 16 CTAs may become resident while the tile
    // kernel is still running; they wait here until its memory is complete and visible.  No-op in plain stream order.
    cudaGridDependencySynchronize();
    sum_split_rows<T>(a, a.s.a(), a.s.b(), /*whole_grid=*/true);
}

// Plain stream order by default.  B200SPMV_PDL=1 opts into programmatic stream serialization (the fix-up CTAs become
// resident while the tile kernel drains).  It is opt-in because one 4-GPU run next to NCCL kernels hung with it and the
// cause was never established.
template <typename T>
static cudaError_t launch_fixup(const CsrArgs<T>& a, cudaStream_t stream) {
    if (a.pdl) {
        cudaLaunchConfig_t cfg = {};
        cfg.gridDim = dim3(16);
        cfg.blockDim = dim3(256);
        cfg.dynamicSmemBytes = 0;
        cfg.stream = stream;
        cudaLaunchAttribute attr[1];
        attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
        attr[0].val.programmaticStreamSerializationAllowed = 1;
        cfg.attrs = attr;
        cfg.numAttrs = 1;
        if (cudaLaunchKernelEx(&cfg, csr_fixup_kernel<T>, a) == cudaSuccess) return cudaSuccess;
        (void)cudaGetLastError();                             // the attribute was refused: fall through to plain order
    }
    csr_fixup_kernel<T><<<16, 256, 0, stream>>>(a);
    return cudaGetLastError();
}


// ================================================================================================
// Persistent, software-pipelined variant (the default): each CTA walks tiles b, b+grid, b+2*grid, ...
// While it reduces tile i out of shared memory (phase 2), the val/col/rowOff loads of tile i+1 are
// already in flight into registers, so the HBM latency of the stream never sits on a tile's critical
// path; what remains per tile is one L2 round trip for the x gathers plus the shared-memory work.
// No CTA launch gaps either: the grid is SMs x (resident CTAs per SM).
// ================================================================================================
constexpr int PIPE_STEPS = B200_CSR_PIPE_STEPS;   // load steps held in registers for the next tile
constexpr int PIPE_OFFS  = B200_CSR_PIPE_OFFS;    // rowOff entries per thread held in registers

template <typename T>
struct TileRegs {
    int c[PIPE_STEPS];
    T   v[PIPE_STEPS];
    int o[PIPE_OFFS];
};

template <typename T>
__device__ __forceinline__ void pipe_issue_loads(const CsrArgs<T>& a, int2 st, int2 en, TileRegs<T>& t) {
    const int rs = st.x, ns = st.y, re = en.x, ne = en.y;
    const int noff = re - rs + 1;
#pragma unroll
    for (int j = 0; j < PIPE_OFFS; j++) {
        const int i = j * CSR_BLOCK + (int)threadIdx.x;
        t.o[j] = i < noff ? __ldg(a.off + rs + i) : 0;
    }
    const int al = ns & ~31, lead = ns - al, span = ne - al;
    const int* colp = a.col + al;
    const T*   valp = a.val + al;
#pragma unroll
    for (int k = 0; k < PIPE_STEPS; k++) {
        const int e = k * CSR_BLOCK + (int)threadIdx.x;
        const bool live = e >= lead && e < span;
        t.c[k] = live ? ldg_stream(colp + e) : a.base;
        t.v[k] = live ? ldg_stream(valp + e) : T(0);
    }
}

template <typename T>
__global__ void __launch_bounds__(CSR_BLOCK, B200_PIPE_MIN_CTAS) csr_pipe_kernel(const CsrArgs<T> a, int num_tiles) {
    __shared__ T   sP[CSR_SMEM_ELEMS];
    __shared__ soff_t sOff[CSR_SMEM_ELEMS + 1];
    __shared__ T   sRed[CSR_BLOCK / 32];

    int b = blockIdx.x;                      // the launcher guarantees gridDim.x <= num_tiles
    const T alpha = a.s.a(), beta = a.s.b();
    int2 st = a.plan.tiles[b], en = a.plan.tiles[b + 1];
    TileRegs<T> t;
    pipe_issue_loads(a, st, en, t);

    for (;;) {
        const int rs = st.x, ns = st.y, re = en.x, ne = en.y;
        TRACE_STAMP(a, b, 0); TRACE_SMID(a, b);
        const int nb = b + (int)gridDim.x;
        const bool has_next = nb < num_tiles;
        int2 nst = st, nen = en;
        if (has_next) { nst = a.plan.tiles[nb]; nen = a.plan.tiles[nb + 1]; }   // descriptor of the next tile, early

        // rowOff slice -> shared memory (rebased to the tile)
        const int noff = re - rs + 1;
#pragma unroll
        for (int j = 0; j < PIPE_OFFS; j++) {
            const int i = j * CSR_BLOCK + (int)threadIdx.x;
            if (i < noff) sOff[i] = to_soff(t.o[j] - a.base - ns);
        }
        for (int i = PIPE_OFFS * CSR_BLOCK + (int)threadIdx.x; i < noff; i += CSR_BLOCK)      // very row-dense tiles only
            sOff[i] = to_soff(__ldg(a.off + rs + i) - a.base - ns);

        // gathers + products
        const int al = ns & ~31, lead = ns - al, span = ne - al;
        {
            T xv[PIPE_STEPS];
#pragma unroll
            for (int k = 0; k < PIPE_STEPS; k++) {
                const int e = k * CSR_BLOCK + (int)threadIdx.x;
                const bool live = e >= lead && e < span;
                xv[k] = (live && !(B200_CSR_ABLATE & 2)) ? __ldg(a.x + (t.c[k] - a.base)) : T(0);
            }
#pragma unroll
            for (int k = 0; k < PIPE_STEPS; k++) {
                const int e = k * CSR_BLOCK + (int)threadIdx.x;
                if (e >= lead && e < span) sP[e - lead] = t.v[k] * xv[k];
            }
        }
        for (int e = PIPE_STEPS * CSR_BLOCK + (int)threadIdx.x; e < span; e += CSR_BLOCK) {   // oversized tiles only
            const int c = ldg_stream(a.col + al + e);
            const T   v = ldg_stream(a.val + al + e);
            sP[e - lead] = v * __ldg(a.x + (c - a.base));
        }
        __syncthreads();
        TRACE_STAMP(a, b, 1);

        if (has_next) pipe_issue_loads(a, nst, nen, t);   // block-uniform; overlaps phase 2 below

        tile_phase2<T, soff_t, CSR_BLOCK, 0>(a, b, rs, ns, re, ne, sP, sOff, 0, sRed, alpha, beta, (int)threadIdx.x);
        TRACE_STAMP(a, b, 2);
        if (!has_next) break;
        __syncthreads();                                   // sP / sOff are free again
        b = nb; st = nst; en = nen;
    }
    split_rows_fixup<T>(a, alpha, beta);
}

// ================================================================================================
// Warp-specialised, TMA-fed variant (B200_CSR_KERNEL == 2).
//
// Measured on the tile / pipe kernels: the three costs of a tile -- streaming val/col from HBM, gathering x through
// L1TEX, reducing the products out of shared memory -- ADD UP when one set of warps performs them one after the
// other, although they use different resources.
// Here each resource gets its own agents inside one persistent CTA, decoupled by a ring of STAGES tile buffers in
// shared memory and mbarriers:
//
//   producer warp   : cp.async.bulk (TMA, 1-D) of the tile's col_ind / val / rowOff slices global -> shared,
//                     complete_tx on full[s].  Runs STAGES tiles ahead:
//                     HBM stays busy no matter what the other warps wait for.
//   gather warps    : wait full[s]; read col from shared, gather x (the only L1TEX-heavy part), multiply with val
//                     from shared, store the product in place; arrive on prod[s].
//   reduce groups   : RGROUPS groups of RWARPS warps, tile i belongs to group i % RGROUPS; wait prod[s]; per-row
//                     reduction out of shared memory (same code as the other kernels), write y; arrive on empty[s].
// ================================================================================================
#ifndef B200_WS_GATHER_WARPS
#define B200_WS_GATHER_WARPS 8
#endif
#ifndef B200_WS_REDUCE_WARPS
#define B200_WS_REDUCE_WARPS 4
#endif
#ifndef B200_WS_REDUCE_GROUPS
#define B200_WS_REDUCE_GROUPS 2
#endif
#ifndef B200_WS_STAGES
#define B200_WS_STAGES 4
#endif
#ifndef B200_WS_MIN_CTAS
#define B200_WS_MIN_CTAS 1
#endif
#ifndef B200_WS_GATHER_UNROLL
#define B200_WS_GATHER_UNROLL 8
#endif
constexpr int WS_GW = B200_WS_GATHER_WARPS, WS_RW = B200_WS_REDUCE_WARPS, WS_RG = B200_WS_REDUCE_GROUPS;
constexpr int WS_STAGES = B200_WS_STAGES;
constexpr int WS_THREADS = 32 * (1 + WS_GW + WS_RW * WS_RG);
constexpr int WS_ELEMS = (CSR_SMEM_ELEMS + 32 + 3) & ~3;        // a tile's [al, ne) range: < SMEM_ELEMS + 32 elements
constexpr int WS_OFFS  = (CSR_SMEM_ELEMS + 1 + 3 + 3) & ~3;     // rowOff[rs&~3 .. re]: <= SMEM_ELEMS + 3 entries

template <typename T>
struct WsStage {
    static constexpr size_t col_bytes = (size_t)WS_ELEMS * sizeof(int);
    static constexpr size_t val_bytes = (size_t)WS_ELEMS * sizeof(T);
    static constexpr size_t off_bytes = (size_t)WS_OFFS * sizeof(int);
    static constexpr size_t bytes = (col_bytes + val_bytes + off_bytes + 127) / 128 * 128;
};

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
    uint32_t ok;
    asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
                 : "=r"(ok) : "r"(smem_u32(bar)), "r"(parity) : "memory");
    return ok != 0;
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    if (mbar_try_wait(bar, parity)) return;
    const long long t0 = clock64();
    while (!mbar_try_wait(bar, parity)) {
        if (clock64() - t0 > 4000000000LL) __trap();   // ~2 s: a protocol bug must not hang the GPU
    }
}
__device__ __forceinline__ void tma_bulk_g2s(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(smem_u32(dst)), "l"(src), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}

template <typename T>
__global__ void __launch_bounds__(WS_THREADS, B200_WS_MIN_CTAS) csr_ws_kernel(const CsrArgs<T> a, int num_tiles) {
    extern __shared__ __align__(128) unsigned char ws_smem[];
    __shared__ uint64_t bar_full[WS_STAGES], bar_off[WS_STAGES], bar_prod[WS_STAGES], bar_empty[WS_STAGES];
    __shared__ T sRed[WS_RG][WS_RW];

    const int tid = (int)threadIdx.x, warp = tid >> 5, lane = tid & 31;
    if (tid == 0) {
#pragma unroll
        for (int s = 0; s < WS_STAGES; s++) {
            mbar_init(&bar_full[s], 1);        // producer's arrive.expect_tx (+ the TMA bytes)
            mbar_init(&bar_off[s], 1);         // producer, after the rowOff slice is in shared memory
            mbar_init(&bar_prod[s], WS_GW);    // one arrive per gather warp
            mbar_init(&bar_empty[s], WS_RW);   // one arrive per warp of the reduce group that owned the tile
        }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    }
    __syncthreads();
    const T alpha = a.s.a(), beta = a.s.b();

    auto stage_col = [&](int s) { return (int*)(ws_smem + (size_t)s * WsStage<T>::bytes); };
    auto stage_val = [&](int s) { return (T*)(ws_smem + (size_t)s * WsStage<T>::bytes + WsStage<T>::col_bytes); };
    auto stage_off = [&](int s) {
        return (int*)(ws_smem + (size_t)s * WsStage<T>::bytes + WsStage<T>::col_bytes + WsStage<T>::val_bytes);
    };

    if (warp == 0) {
        // ------------------------------------------------ producer ------------------------------------------------
        int i = 0;
        for (int b = blockIdx.x; b < num_tiles; b += gridDim.x, i++) {
            const int s = i % WS_STAGES, n = i / WS_STAGES;
            if (n > 0) mbar_wait(&bar_empty[s], (uint32_t)((n - 1) & 1));
            const int2 st = a.plan.tiles[b], en = a.plan.tiles[b + 1];
            const int rs = st.x, ns = st.y, re = en.x, ne = en.y;
            const int al = ns & ~31, span = ne - al;
            int copied = (span + 3) & ~3;                       // whole 16-byte units ...
            if (copied > a.nnz - al) copied = (a.nnz - al) & ~3;  // ... that stay inside the arrays
            // rowOff[rs4 .. re] (rs4 = rs rounded down to a 16-byte boundary), raw values
            const int rs4 = rs & ~3;
            int ocopied = (re - rs4 + 1 + 3) & ~3;
            if (ocopied > a.rows + 1 - rs4) ocopied = (a.rows + 1 - rs4) & ~3;
            int* so = stage_off(s);
            if (lane == 0) {
                asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
                mbar_arrive_expect_tx(&bar_full[s], (uint32_t)(copied * (sizeof(int) + sizeof(T)) + ocopied * sizeof(int)));
                if (copied > 0) {
                    tma_bulk_g2s(stage_col(s), a.col + al, (uint32_t)(copied * sizeof(int)), &bar_full[s]);
                    tma_bulk_g2s(stage_val(s), a.val + al, (uint32_t)(copied * sizeof(T)), &bar_full[s]);
                }
                if (ocopied > 0) tma_bulk_g2s(so, a.off + rs4, (uint32_t)(ocopied * sizeof(int)), &bar_full[s]);
            }
            for (int j = ocopied + lane; j < re - rs4 + 1; j += 32) so[j] = __ldg(a.off + rs4 + j);   // <= 3 entries, last tile only
            __syncwarp();
            if (lane == 0) mbar_arrive(&bar_off[s]);
        }
    } else if (warp <= WS_GW) {
        // ------------------------------------------------ gather warps --------------------------------------------
        const int gtid = tid - 32;
        constexpr int GT = WS_GW * 32, UNR = B200_WS_GATHER_UNROLL;
        int i = 0;
        for (int b = blockIdx.x; b < num_tiles; b += gridDim.x, i++) {
            const int s = i % WS_STAGES, n = i / WS_STAGES;
            const int2 st = a.plan.tiles[b], en = a.plan.tiles[b + 1];
            const int ns = st.y, ne = en.y;
            const int al = ns & ~31, lead = ns - al, span = ne - al;
            int copied = (span + 3) & ~3;
            if (copied > a.nnz - al) copied = (a.nnz - al) & ~3;
            const int* sc = stage_col(s);
            T*         sv = stage_val(s);
            mbar_wait(&bar_full[s], (uint32_t)(n & 1));
            for (int e0 = 0; e0 < span; e0 += GT * UNR) {
                int c[UNR];
                T   xv[UNR];
#pragma unroll
                for (int u = 0; u < UNR; u++) {
                    const int e = e0 + u * GT + gtid;
                    const bool live = e >= lead && e < span;
                    c[u] = !live ? a.base : (e < copied ? sc[e] : ldg_stream(a.col + al + e));
                }
#pragma unroll
                for (int u = 0; u < UNR; u++) {
                    const int e = e0 + u * GT + gtid;
                    const bool live = e >= lead && e < span;
                    xv[u] = (live && !(B200_CSR_ABLATE & 2)) ? __ldg(a.x + (c[u] - a.base)) : T(0);
                }
#pragma unroll
                for (int u = 0; u < UNR; u++) {
                    const int e = e0 + u * GT + gtid;
                    if (e >= lead && e < span) {
                        const T v = e < copied ? sv[e] : ldg_stream(a.val + al + e);
                        sv[e] = v * xv[u];
                    }
                }
            }
            __syncwarp();
            if (lane == 0) mbar_arrive(&bar_prod[s]);
        }
    } else {
        // ------------------------------------------------ reduce groups -------------------------------------------
        const int rwarp = warp - 1 - WS_GW;                 // 0 .. RW*RG-1
        const int grp = rwarp / WS_RW, rtid = tid - 32 * (1 + WS_GW) - grp * (WS_RW * 32);
        int i = 0;
        for (int b = blockIdx.x; b < num_tiles; b += gridDim.x, i++) {
            if (i % WS_RG != grp) continue;
            const int s = i % WS_STAGES, n = i / WS_STAGES;
            const int2 st = a.plan.tiles[b], en = a.plan.tiles[b + 1];
            const int rs = st.x, ns = st.y, re = en.x, ne = en.y;
            const int lead = ns - (ns & ~31);
            mbar_wait(&bar_off[s], (uint32_t)(n & 1));
            mbar_wait(&bar_full[s], (uint32_t)(n & 1));
            mbar_wait(&bar_prod[s], (uint32_t)(n & 1));
            const int* so = stage_off(s) + (rs - (rs & ~3));
            const int shift = a.base + ns;
            if (grp == 0)
                tile_phase2<T, int, WS_RW * 32, 1>(a, b, rs, ns, re, ne, stage_val(s) + lead, so, shift, sRed[0], alpha, beta, rtid);
            else if (grp == 1)
                tile_phase2<T, int, WS_RW * 32, 2>(a, b, rs, ns, re, ne, stage_val(s) + lead, so, shift, sRed[WS_RG > 1 ? 1 : 0], alpha, beta, rtid);
            else if (grp == 2)
                tile_phase2<T, int, WS_RW * 32, 3>(a, b, rs, ns, re, ne, stage_val(s) + lead, so, shift, sRed[WS_RG > 2 ? 2 : 0], alpha, beta, rtid);
            else
                tile_phase2<T, int, WS_RW * 32, 4>(a, b, rs, ns, re, ne, stage_val(s) + lead, so, shift, sRed[WS_RG > 3 ? 3 : 0], alpha, beta, rtid);
            __syncwarp();
            if (lane == 0) mbar_arrive(&bar_empty[s]);
        }
    }
    split_rows_fixup<T>(a, alpha, beta);
}

// ================================================================================================
// Row-wise variant (B200_CSR_KERNEL == 3): the tile partition bounds and balances the work, but inside a tile the
// products never touch shared memory.  A group of G lanes (G picked per tile from its mean row length) owns ROWS rows
// at a time: it reads their val/col segments straight from global memory (neighbouring groups own neighbouring rows,
// so a warp-level load still covers one contiguous span), gathers x, accumulates in registers and finishes with one
// shuffle tree per row.  Rationale (measured): the SM's L1TEX pipe is the bottleneck resource on scattered matrices
// and serves gathers, shared-memory accesses and shuffles strictly one after the other, so every STS/LDS of a product
// costs as much as a gather; this variant spends the pipe on gathers + log2(G) shuffles per ROW only.
// ================================================================================================
#ifndef B200_RW_ROWS
#define B200_RW_ROWS 4
#endif
#ifndef B200_RW_U
#define B200_RW_U 2
#endif

template <typename T, int G, int ROWS, int U, int BLOCK>
__device__ __forceinline__ void rowwise_rows(const CsrArgs<T>& a, int r_first, int nrows, T alpha, T beta, int tid) {
    constexpr int GROUPS = BLOCK / G;
    const int gid = tid / G, gl = tid % G;
    const int* off = a.off + r_first;
    const int* colp = a.col - a.base;     // off[] values are base-indexed positions
    const T*   valp = a.val - a.base;
    const T*   xp   = a.x - a.base;
    for (int r0 = 0; r0 < nrows; r0 += GROUPS * ROWS) {
        int k0[ROWS], e[ROWS];
#pragma unroll
        for (int i = 0; i < ROWS; i++) {
            const int ri = r0 + i * GROUPS + gid;
            const bool active = ri < nrows;
            k0[i] = (active ? __ldg(off + ri) : 0) + gl;
            e[i]  = active ? __ldg(off + ri + 1) : 0;
        }
        int c[ROWS][U];
        T   v[ROWS][U];
#pragma unroll
        for (int i = 0; i < ROWS; i++)
#pragma unroll
            for (int u = 0; u < U; u++) {
                const int k = k0[i] + u * G;
                const bool live = k < e[i];
                c[i][u] = live ? ldg_stream(colp + k) : a.base;
                v[i][u] = live ? ldg_stream(valp + k) : T(0);
            }
        T sum[ROWS];
#pragma unroll
        for (int i = 0; i < ROWS; i++) {
            T xv[U];
#pragma unroll
            for (int u = 0; u < U; u++) xv[u] = (k0[i] + u * G < e[i]) ? __ldg(xp + c[i][u]) : T(0);
            sum[i] = v[i][0] * xv[0];
#pragma unroll
            for (int u = 1; u < U; u++) sum[i] += v[i][u] * xv[u];
        }
#pragma unroll
        for (int i = 0; i < ROWS; i++) {                        // rows longer than U*G: batches of U loads in flight
            for (int kb = k0[i] + U * G; kb < e[i]; kb += U * G) {
                int cc[U];
                T   vv[U], xx[U];
#pragma unroll
                for (int u = 0; u < U; u++) {
                    const bool live = kb + u * G < e[i];
                    cc[u] = live ? ldg_stream(colp + kb + u * G) : a.base;
                    vv[u] = live ? ldg_stream(valp + kb + u * G) : T(0);
                }
#pragma unroll
                for (int u = 0; u < U; u++) xx[u] = (kb + u * G < e[i]) ? __ldg(xp + cc[u]) : T(0);
#pragma unroll
                for (int u = 0; u < U; u++) sum[i] += vv[u] * xx[u];
            }
        }
        if (ROWS == 4 && G >= 4) {
            // Transposed butterfly: 4 row sums over G lanes in 2 + 1 + log2(G/4) exchanges instead of 4*log2(G)
            // (shuffles queue in the same L1TEX pipe as the gathers).  After the first two exchanges every lane of
            // quarter q = 2*hi + mid of the group carries one partial of row slot q.
            const bool hi = (gl & (G / 2)) != 0, mid = (gl & (G / 4)) != 0;
            const T s0 = hi ? sum[0] : sum[2], s1 = hi ? sum[1] : sum[3];
            T k0v = (hi ? sum[2] : sum[0]) + __shfl_xor_sync(0xffffffffu, s0, G / 2);
            T k1v = (hi ? sum[3] : sum[1]) + __shfl_xor_sync(0xffffffffu, s1, G / 2);
            T kv  = (mid ? k1v : k0v) + __shfl_xor_sync(0xffffffffu, mid ? k0v : k1v, G / 4);
#pragma unroll
            for (int o = G / 8; o > 0; o >>= 1) kv += __shfl_xor_sync(0xffffffffu, kv, o);
            if ((gl & (G / 4 - 1)) == 0) {
                const int slot = (hi ? 2 : 0) + (mid ? 1 : 0);
                const int ri = r0 + slot * GROUPS + gid;
                if (ri < nrows) {
                    T* yp = a.y + r_first + ri;
                    *yp = axpby(alpha, kv, beta, yp);
                }
            }
        } else {
#pragma unroll
            for (int o = G / 2; o > 0; o >>= 1)
#pragma unroll
                for (int i = 0; i < ROWS; i++) sum[i] += __shfl_down_sync(0xffffffffu, sum[i], o, G);
            if (gl == 0) {
#pragma unroll
                for (int i = 0; i < ROWS; i++) {
                    const int ri = r0 + i * GROUPS + gid;
                    if (ri < nrows) {
                        T* yp = a.y + r_first + ri;
                        *yp = axpby(alpha, sum[i], beta, yp);
                    }
                }
            }
        }
    }
}

// Sum val[k]*x[col[k]] for k in [lo, hi) (0-based positions) with the whole CTA; result valid on thread 0.
template <typename T, int BLOCK>
__device__ __forceinline__ T block_dot_range(const CsrArgs<T>& a, int lo, int hi, T* sRed, int tid) {
    T s = T(0);
    for (int k = lo + tid; k < hi; k += 4 * BLOCK) {
        int cc[4];
        T   vv[4];
#pragma unroll
        for (int u = 0; u < 4; u++) {
            const bool live = k + u * BLOCK < hi;
            cc[u] = live ? ldg_stream(a.col + k + u * BLOCK) : a.base;
            vv[u] = live ? ldg_stream(a.val + k + u * BLOCK) : T(0);
        }
#pragma unroll
        for (int u = 0; u < 4; u++) s += (k + u * BLOCK < hi) ? vv[u] * __ldg(a.x + (cc[u] - a.base)) : T(0);
    }
    s = warp_sum(s);
    __syncthreads();
    if ((tid & 31) == 0) sRed[tid >> 5] = s;
    __syncthreads();
    T tot = T(0);
    if (tid == 0) {
#pragma unroll
        for (int w = 0; w < BLOCK / 32; w++) tot += sRed[w];
    }
    return tot;
}

template <typename T>
__global__ void __launch_bounds__(CSR_BLOCK, B200_RW_MIN_CTAS) csr_rowwise_kernel(const CsrArgs<T> a) {
    __shared__ T sRed[CSR_BLOCK / 32];
    const int  b  = blockIdx.x, tid = (int)threadIdx.x;
    const int2 st = a.plan.tiles[b], en = a.plan.tiles[b + 1];
    const int  rs = st.x, ns = st.y, re = en.x, ne = en.y;
    const T alpha = a.s.a(), beta = a.s.b();
    if (a.pdl) cudaTriggerProgrammaticLaunchCompletion();

    bool head = false;
    int  head_end = ns;                      // non-zeros [ns, head_end) belong to the split row rs
    if (rs < a.rows && ns > __ldg(a.off + rs) - a.base) {
        head = true;
        const int o1 = __ldg(a.off + rs + 1) - a.base;
        head_end = o1 < ne ? o1 : ne;
    }
    const int r_first = rs + (head ? 1 : 0);
    const int nrows   = re - r_first;
    bool tail = false;
    int  tail_beg = ne;                      // non-zeros [tail_beg, ne) belong to the split row re
    if (re < a.rows && re >= r_first) {
        const int o0 = __ldg(a.off + re) - a.base;
        if (ne > o0) { tail = true; tail_beg = o0; }
    }
    if (nrows > 0) {
        const int body = tail_beg - head_end;
        const int avg2 = body / (2 * nrows);
        if      (avg2 <= 1)  rowwise_rows<T, 1,  B200_RW_ROWS, B200_RW_U, CSR_BLOCK>(a, r_first, nrows, alpha, beta, tid);
        else if (avg2 <= 2)  rowwise_rows<T, 2,  B200_RW_ROWS, B200_RW_U, CSR_BLOCK>(a, r_first, nrows, alpha, beta, tid);
        else if (avg2 <= 4)  rowwise_rows<T, 4,  B200_RW_ROWS, B200_RW_U, CSR_BLOCK>(a, r_first, nrows, alpha, beta, tid);
        else if (avg2 <= 8)  rowwise_rows<T, 8,  B200_RW_ROWS, B200_RW_U, CSR_BLOCK>(a, r_first, nrows, alpha, beta, tid);
        else if (avg2 <= 16) rowwise_rows<T, 16, B200_RW_ROWS, B200_RW_U, CSR_BLOCK>(a, r_first, nrows, alpha, beta, tid);
        else                 rowwise_rows<T, 32, 2, 4, CSR_BLOCK>(a, r_first, nrows, alpha, beta, tid);
    }
    if (head) {
        const T hs = block_dot_range<T, CSR_BLOCK>(a, ns, head_end, sRed, tid);
        if (tid == 0) a.plan.head_part[b] = (double)hs;
    }
    if (tail) {
        const T ts = block_dot_range<T, CSR_BLOCK>(a, tail_beg, ne, sRed, tid);
        if (tid == 0) a.plan.tail_part[b] = (double)ts;
    }
}

// SMs x resident CTAs per SM of a kernel on the current device (cached per device / kernel, thread-safe).
static int resident_ctas(const void* kernel, int block = CSR_BLOCK, size_t dyn_smem = 0) {
    struct Entry { int dev; const void* k; int n; };
    static Entry cache[64];
    static int ncache = 0;
    static std::mutex mu;
    int dev = 0;
    cudaGetDevice(&dev);
    std::lock_guard<std::mutex> lk(mu);
    for (int i = 0; i < ncache; i++)
        if (cache[i].dev == dev && cache[i].k == kernel) return cache[i].n;
    int sms = 132, per = 1;
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    if (dyn_smem > 48 * 1024) cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)dyn_smem);
    cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per, kernel, block, dyn_smem);
    if (per < 1) per = 1;
    const int n = sms * per;
    if (ncache < 64) cache[ncache++] = Entry{dev, kernel, n};
    return n;
}

template <typename T>
static int launch_csr(cudaStream_t stream, int64_t rows, int64_t nnz, const void* off, const void* col,
                      const void* val, int base, const void* alpha, const void* beta, int on_device,
                      const void* x, void* y, void* ws) {
    const int64_t nt = csr_num_tiles(rows, nnz);
    if (nt == 0) return 0;
    const Config& cf = config();
    CsrArgs<T> a;
    a.off = (const int*)off; a.col = (const int*)col; a.val = (const T*)val;
    a.x = (const T*)x; a.y = (T*)y; a.base = base; a.rows = (int)rows; a.nnz = (int)nnz;
    set_scalars(a.s, alpha, beta, on_device);
    plan_layout(nt, ws, &a.plan);
    a.trace = nullptr;
    a.num_tiles = (unsigned)nt;
    a.tile_stride = 1;
    a.seg_dense = cf.seg_dense;
    a.pdl = cf.pdl;
    if (cf.tile_scatter && nt > 2) {                  // stride ~ 0.618 * nt, coprime with nt -> a permutation of the tiles
        auto gcd = [](uint64_t x, uint64_t y) { while (y) { uint64_t t = x % y; x = y; y = t; } return x; };
        uint64_t st = (uint64_t)(0.6180339887 * (double)nt) | 1;
        while (gcd(st, (uint64_t)nt) != 1) st += 2;
        a.tile_stride = (unsigned)(st % (uint64_t)nt);
    }
#ifdef B200_CSR_TRACE
    a.trace = g_trace_ptr;
#endif
    // Which kernel?  Matrices with short rows (stencils, < 12 non-zeros per row on
    // average) run fastest on the persistent software-pipelined kernel; longer / skewed rows on one CTA per tile with
    // register accumulation (seg).  B200SPMV_CSR_KERNEL=tile|pipe|ws|rowwise|seg (or b200spmv_set_option) overrides,
    // as does -DB200_CSR_KERNEL at build time.
    int mode = B200_CSR_KERNEL;
    if (mode < 0) mode = cf.csr_kernel >= 0 ? cf.csr_kernel : (nnz >= 12 * rows ? 0 : 1);
    if (mode == 2 && (((uintptr_t)col | (uintptr_t)val | (uintptr_t)off) & 15) != 0) mode = 1;   // TMA needs 16 B alignment
    cudaError_t err = cudaSuccess;
    constexpr bool F64 = sizeof(T) == 8;
    stats().last_csr_kernel = mode == 0 ? (F64 ? "b200::csr_tile_kernel<double>" : "b200::csr_tile_kernel<float>")
                            : mode == 5 ? (F64 ? "b200::csr_seg_kernel<double>" : "b200::csr_seg_kernel<float>")
                            : mode == 3 ? (F64 ? "b200::csr_rowwise_kernel<double>" : "b200::csr_rowwise_kernel<float>")
                            : mode == 2 ? (F64 ? "b200::csr_ws_kernel<double>" : "b200::csr_ws_kernel<float>")
                                        : (F64 ? "b200::csr_pipe_kernel<double>" : "b200::csr_pipe_kernel<float>");
    if (mode == 0 || mode == 3 || mode == 5) {
        if (mode == 0)      csr_tile_kernel<T><<<(unsigned)nt, CSR_BLOCK, 0, stream>>>(a);
        else if (mode == 5) csr_seg_kernel<T><<<(unsigned)nt, CSR_BLOCK, 0, stream>>>(a);
        else                csr_rowwise_kernel<T><<<(unsigned)nt, CSR_BLOCK, 0, stream>>>(a);
        err = cudaGetLastError();                      // a failed main launch must not be masked by the fix-up launch
        if (err == cudaSuccess) err = launch_fixup<T>(a, stream);
    } else if (mode == 2) {
        const size_t dyn = (size_t)WS_STAGES * WsStage<T>::bytes;
        int64_t grid = (int64_t)resident_ctas((const void*)csr_ws_kernel<T>, WS_THREADS, dyn);
        if (grid > nt) grid = nt;
        csr_ws_kernel<T><<<(unsigned)grid, WS_THREADS, dyn, stream>>>(a, (int)nt);
        err = cudaGetLastError();
    } else {
        int64_t grid = (int64_t)resident_ctas((const void*)csr_pipe_kernel<T>);
        if (grid > nt) grid = nt;
        csr_pipe_kernel<T><<<(unsigned)grid, CSR_BLOCK, 0, stream>>>(a, (int)nt);
        err = cudaGetLastError();
    }
    return (int)err;
}

}  // namespace b200

using namespace b200;

extern "C" {

size_t b200spmv_csr_workspace_bytes(int64_t rows, int64_t nnz) {
    if (rows < 0 || nnz < 0) return 0;
    return plan_layout(csr_num_tiles(rows, nnz), nullptr, nullptr);
}

int64_t b200spmv_csr_num_tiles(int64_t rows, int64_t nnz) { return csr_num_tiles(rows, nnz); }

void b200spmv_csr_plan_params(int32_t* tile_items, int32_t* long_row, int32_t* block_threads) {
    if (tile_items) *tile_items = CSR_TILE_ITEMS;
    if (long_row) *long_row = CSR_LONG_ROW;
    if (block_threads) *block_threads = CSR_BLOCK;
}

size_t b200spmv_csr_plan_tiles_offset(void) { return PLAN_HEADER_BYTES; }

size_t b200spmv_csr_plan_ctl_offset(int64_t rows, int64_t nnz) {
    PlanView v;
    plan_layout(csr_num_tiles(rows, nnz), nullptr, &v);
    return (size_t)((char*)v.ctl - (char*)nullptr);
}

size_t b200spmv_csr_plan_split_offset(int64_t rows, int64_t nnz) {
    PlanView v;
    plan_layout(csr_num_tiles(rows, nnz), nullptr, &v);
    return (size_t)((char*)v.split - (char*)nullptr);
}

int b200spmv_csr_analyze(void* stream, int64_t rows, int64_t nnz, const void* row_offsets, int32_t base,
                         void* workspace) {
    if (rows < 0 || nnz < 0 || rows > INT32_MAX - 1 || nnz > INT32_MAX - 1 || !workspace || (rows > 0 && !row_offsets))
        return -1;
    const int64_t nt = csr_num_tiles(rows, nnz);
    PlanView v;
    plan_layout(nt, workspace, &v);
    if (rows == 0) return 0;  // (the first PLAN_HEADER_BYTES of the workspace are reserved, unused on device)
    cudaError_t e = cudaMemsetAsync(v.ctl, 0, 64, (cudaStream_t)stream);
    if (e != cudaSuccess) return (int)e;
    const int threads = 128;
    const unsigned blocks = (unsigned)((nt + 1 + threads - 1) / threads);
    csr_partition_kernel<<<blocks, threads, 0, (cudaStream_t)stream>>>((const int*)row_offsets, base, rows, nnz, nt, v);
    return (int)cudaGetLastError();
}

int b200spmv_csr_mv(void* stream, int dtype, int64_t rows, int64_t cols, int64_t nnz, const void* row_offsets,
                    const void* col_ind, const void* values, int32_t base, const void* alpha, const void* beta,
                    int scalars_on_device, const void* x, void* y, void* workspace) {
    if (rows < 0 || cols < 0 || nnz < 0 || !alpha || !beta) return -1;
    if (rows == 0) return 0;
    if (!row_offsets || !y || !workspace || (nnz > 0 && (!col_ind || !values || !x))) return -1;
    if (dtype == 0)
        return launch_csr<float>((cudaStream_t)stream, rows, nnz, row_offsets, col_ind, values, base, alpha, beta,
                                 scalars_on_device, x, y, workspace);
    if (dtype == 1)
        return launch_csr<double>((cudaStream_t)stream, rows, nnz, row_offsets, col_ind, values, base, alpha, beta,
                                  scalars_on_device, x, y, workspace);
    return -1;
}

}  // extern "C"
