// spmm_coo.cu -- COO x dense  C = alpha * op(A) * B + beta * C  on H100 (sm_90a), fp32 / fp64, int32 indices, strided batches.
// Replaces the closed library behind cusparseSpMM for COO descriptors (cuSPARSE/spmm_coo/spmm_coo_example.c:110-122,
// cuSPARSE/spmm_coo_batched/spmm_coo_batched_example.c:137-162).
//
// The work is split by non-zero count, not by row: warp w owns SPMM_COO_CHUNK consecutive entries and one panel of 64 columns of
// B / C (two per lane, as spmm_csr_kernel).  (row, col, val) are loaded 32 at a time with one coalesced instruction each and
// broadcast by shuffle; runs of equal row index are accumulated in registers.  A hub row of R-MAT is spread over as many warps as
// it has chunks, where spmm_csr_kernel gives it one warp.
//
// Two paths, both launched on every call; each reads a per-batch "unsorted" flag in the workspace and returns at once when the
// call is not its case, so there is no host synchronisation, no allocation, and the call can be captured in a CUDA graph:
//   * spmm_coo_check_kernel sets the flag on any descending pair of row indices (the flag is reset by cudaMemsetAsync first).
//   * Row-sorted A (flag clear): deterministic, no atomics.  A run wholly inside a chunk writes its C row once
//     (alpha * acc + beta * C).  Each chunk's first and last runs go to two carry slots in the workspace; spmm_coo_fixup_kernel
//     adds the carries of a row in ascending chunk order and writes that row once, however many chunks the row spans.  Rows that
//     store nothing get beta * C (0 for beta == 0, C not read): the chunk whose first entry follows such a gap writes it, chunk 0
//     the rows before the first entry, the last chunk the rows behind the last entry.  Every entry of C is written exactly once.
//   * Unsorted A (flag set), A^T (the index arrays swapped, as the COO SpMV does), or no usable workspace: spmm_coo_scale_kernel
//     writes C = beta * C, then spmm_coo_atomic_kernel adds alpha * (run sum) with one atomic per run of equal row index and
//     column, as coo_seg_kernel does for SpMV.  Correct for any entry order and for duplicate entries.
// A column-major B is copied row-major into the workspace first (spmm_transpose_b_kernel of spmm_csr.cu, n >= 4, as for CSR).
// A column-major C is written with strided stores.  Lanes past n, ld padding and rows of B no entry references are never read.
#include "spmv_common.cuh"
#include "config.h"
#include "../../include/b200spmv.h"

#include <algorithm>
#include <utility>

namespace b200 {

int transpose_col_to_row_major(cudaStream_t stream, int dtype, const void* B, int64_t ldb, void* Bt, int64_t cols, int64_t n);

#ifndef B200_SPMM_COO_CHUNK
#define B200_SPMM_COO_CHUNK 256
#endif
constexpr int COO_MM_CHUNK = B200_SPMM_COO_CHUNK;   // consecutive non-zeros per warp
constexpr int COO_MM_PANEL = 64;                    // columns of B / C per warp (2 per lane)
constexpr int COO_MM_WARPS = 8;                     // warps per CTA
constexpr int COO_MM_MIN_N_FOR_TRANSPOSE = 4;       // the CSR rule (spmm_csr.cu)
constexpr int COO_MM_STRIDE_CTAS = 132 * 8;         // grid of the grid-stride kernels (check / scale / atomic)
static_assert(COO_MM_CHUNK % 32 == 0, "a chunk is whole 32-entry steps");

template <typename T>
struct CooMmArgs {
    const int* row;
    const int* col;
    const T*   val;
    const T*   B;
    T*         C;
    int        base, rows, n, nnz, nchunks, npanels;
    long long  sbk, sbj, sci, scj;                // B(k, j) = B[k * sbk + j * sbj], C(i, j) = C[i * sci + j * scj]
    long long  a_stride, b_stride, c_stride;      // elements between the matrices of a batch (0 = shared)
    const int* flags;                             // per batch: 1 = unsorted; nullptr = the atomic path unconditionally
    int*       carry_row;                         // [batch][nchunks][2]: row of a chunk's first / last run (-1: none)
    T*         carry_val;                         // [batch][nchunks][npanels][2][64]
    Scalars<T> s;
};

// beta * C, or 0 for beta == 0 without reading C
template <typename T>
__device__ __forceinline__ T scaled(T beta, const T* c) { return beta == T(0) ? T(0) : beta * *c; }

template <typename T>
__device__ __forceinline__ void scale_rows(const CooMmArgs<T>& a, T* C, int lo, int hi, int ja, int jb, bool la, bool lb, T beta) {
    for (int r = lo; r < hi; r++) {
        T* cr = C + (long long)r * a.sci;
        if (la) { T* p = cr + (long long)ja * a.scj; *p = scaled(beta, p); }
        if (lb) { T* p = cr + (long long)jb * a.scj; *p = scaled(beta, p); }
    }
}

// One warp's walk over its chunk [n0, n1) for columns ja / jb: on every change of row index, emit(row, acc0, acc1) for the run
// that ended; returns the row of the last run with its sums in acc0 / acc1.  Warp-uniform control flow: the row index is
// broadcast, so every lane sees the same runs.
template <typename T, typename Emit>
__device__ __forceinline__ int walk_chunk(const CooMmArgs<T>& a, const int* row, const int* col, const T* val, const T* B, int n0,
                                          int n1, int lane, int ja, int jb, bool la, bool lb, T& acc0, T& acc1, Emit emit) {
    const T* Ba = B + (long long)ja * a.sbj;
    const T* Bb = B + (long long)jb * a.sbj;
    int cur = __shfl_sync(0xffffffffu, n0 + lane < n1 ? ldg_stream(row + n0 + lane) - a.base : 0, 0);
    acc0 = T(0); acc1 = T(0);
    for (int p = n0; p < n1; p += 32) {
        const int i = p + lane;
        const bool in = i < n1;
        const int r = in ? ldg_stream(row + i) - a.base : 0;
        const int c = in ? ldg_stream(col + i) - a.base : 0;
        const T   v = in ? ldg_stream(val + i) : T(0);
        const int cnt = min(32, n1 - p);
        for (int t = 0; t < cnt; t += 4) {                       // four B rows in flight per lane
            int rr[4], kk[4];
            T   vv[4], b0[4], b1[4];
#pragma unroll
            for (int u = 0; u < 4; u++) {
                rr[u] = __shfl_sync(0xffffffffu, r, (t + u) & 31);
                kk[u] = __shfl_sync(0xffffffffu, c, (t + u) & 31);
                vv[u] = __shfl_sync(0xffffffffu, v, (t + u) & 31);
            }
#pragma unroll
            for (int u = 0; u < 4; u++) {                        // no entry past cnt: neither a load nor a product
                const long long ro = (long long)kk[u] * a.sbk;
                const bool live = t + u < cnt;
                b0[u] = la && live ? __ldg(Ba + ro) : T(0);
                b1[u] = lb && live ? __ldg(Bb + ro) : T(0);
            }
#pragma unroll
            for (int u = 0; u < 4; u++) {
                if (t + u < cnt) {
                    if (rr[u] != cur) {
                        emit(cur, rr[u], acc0, acc1);
                        cur = rr[u]; acc0 = T(0); acc1 = T(0);
                    }
                    acc0 += vv[u] * b0[u];
                    acc1 += vv[u] * b1[u];
                }
            }
        }
    }
    return cur;
}

// Any descending pair of row indices sets the batch's flag.
__global__ void __launch_bounds__(256) spmm_coo_check_kernel(const int* __restrict__ row, int nnz, long long a_stride, int* flags) {
    const int* r = row + (long long)blockIdx.z * a_stride;
    bool bad = false;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i + 1 < nnz; i += (long long)gridDim.x * blockDim.x)
        bad |= ldg_stream(r + i) > ldg_stream(r + i + 1);
    if (__any_sync(0xffffffffu, bad) && ((int)threadIdx.x & 31) == 0) flags[blockIdx.z] = 1;
}

// Row-sorted path, part 1: interior runs and empty rows straight into C, first / last runs into the carry slots.
template <typename T>
__global__ void __launch_bounds__(32 * COO_MM_WARPS) spmm_coo_sorted_kernel(const CooMmArgs<T> a) {
    const int lane = (int)threadIdx.x & 31;
    const int chunk = blockIdx.x * COO_MM_WARPS + ((int)threadIdx.x >> 5);
    const int bi = blockIdx.z;
    if (chunk >= a.nchunks || a.flags[bi]) return;                 // warp-uniform
    const int* row = a.row + bi * a.a_stride;
    const int* col = a.col + bi * a.a_stride;
    const T*   val = a.val + bi * a.a_stride;
    const T*   B = a.B + bi * a.b_stride;
    T*         C = a.C + bi * a.c_stride;
    const int n0 = chunk * COO_MM_CHUNK, n1 = min(n0 + COO_MM_CHUNK, a.nnz);
    const int panel = blockIdx.y;
    const int ja = panel * COO_MM_PANEL + lane, jb = ja + 32;
    const bool la = ja < a.n, lb = jb < a.n;
    const T alpha = a.s.a(), beta = a.s.b();
    const long long slot0 = (long long)bi * a.nchunks + chunk;     // this chunk's pair of carry rows
    T* carry = a.carry_val + (slot0 * a.npanels + panel) * 2 * COO_MM_PANEL;
    const bool rec = panel == 0 && lane == 0;                       // one lane records the carry rows
    // empty rows in front of the chunk's first entry, behind the previous chunk's last one (chunk 0: from row 0)
    const int prev = n0 > 0 ? ldg_stream(row + n0 - 1) - a.base : -1;
    const int first = ldg_stream(row + n0) - a.base;
    scale_rows(a, C, prev + 1, first, ja, jb, la, lb, beta);
    int runs = 0;
    T acc0, acc1;
    const int last = walk_chunk(a, row, col, val, B, n0, n1, lane, ja, jb, la, lb, acc0, acc1, [&](int r, int next, T s0, T s1) {
        if (runs == 0) {                                            // the chunk's first run: carry slot 0
            if (la) carry[lane] = s0;
            if (lb) carry[32 + lane] = s1;
            if (rec) a.carry_row[slot0 * 2] = r;
        } else {                                                    // wholly inside the chunk: C written once
            T* cr = C + (long long)r * a.sci;
            if (la) { T* p = cr + (long long)ja * a.scj; *p = axpby(alpha, s0, beta, p); }
            if (lb) { T* p = cr + (long long)jb * a.scj; *p = axpby(alpha, s1, beta, p); }
        }
        scale_rows(a, C, r + 1, next, ja, jb, la, lb, beta);       // rows between two runs store nothing
        runs++;
    });
    const int s = runs == 0 ? 0 : 1;                                // the last run: slot 1, or slot 0 when it is also the first
    if (la) carry[s * COO_MM_PANEL + lane] = acc0;
    if (lb) carry[s * COO_MM_PANEL + 32 + lane] = acc1;
    if (rec) {
        a.carry_row[slot0 * 2 + s] = last;
        if (s == 0) a.carry_row[slot0 * 2 + 1] = -1;
    }
    if (chunk == a.nchunks - 1) scale_rows(a, C, last + 1, a.rows, ja, jb, la, lb, beta);
}

// Row-sorted path, part 2: the warp of a row's first carry slot adds all of that row's carries in ascending chunk order and writes
// the row once.  Slot 0 of every chunk holds a run; slot 1 may be empty (-1).
template <typename T>
__global__ void __launch_bounds__(32 * COO_MM_WARPS) spmm_coo_fixup_kernel(const CooMmArgs<T> a) {
    const int lane = (int)threadIdx.x & 31;
    const int q = blockIdx.x * COO_MM_WARPS + ((int)threadIdx.x >> 5);
    const int bi = blockIdx.z;
    if (q >= 2 * a.nchunks || a.flags[bi]) return;                  // warp-uniform
    const int* cr = a.carry_row + (long long)bi * a.nchunks * 2;
    const int r = cr[q];
    if (r < 0) return;
    if (q > 0) {
        const int pq = cr[q - 1] >= 0 ? q - 1 : q - 2;              // q - 1 empty: it is a slot 1, so q - 2 is a slot 0
        if (cr[pq] == r) return;                                     // not the row's first carry
    }
    const int panel = blockIdx.y;
    const int ja = panel * COO_MM_PANEL + lane, jb = ja + 32;
    const bool la = ja < a.n, lb = jb < a.n;
    auto cv = [&](int qq) { return a.carry_val + (((long long)bi * a.nchunks + (qq >> 1)) * a.npanels + panel) * 2 * COO_MM_PANEL +
                                   (qq & 1) * COO_MM_PANEL; };
    T acc0 = la ? cv(q)[lane] : T(0), acc1 = lb ? cv(q)[32 + lane] : T(0);
    for (int qq = q + 1; qq < 2 * a.nchunks; qq++) {
        const int r2 = cr[qq];
        if (r2 < 0) continue;
        if (r2 != r) break;
        if (la) acc0 += cv(qq)[lane];
        if (lb) acc1 += cv(qq)[32 + lane];
    }
    const T alpha = a.s.a(), beta = a.s.b();
    T* crow = a.C + bi * a.c_stride + (long long)r * a.sci;
    if (la) { T* p = crow + (long long)ja * a.scj; *p = axpby(alpha, acc0, beta, p); }
    if (lb) { T* p = crow + (long long)jb * a.scj; *p = axpby(alpha, acc1, beta, p); }
}

// Atomic path, part 1: C = beta * C (0 for beta == 0, C not read), in C's storage order.
template <typename T>
__global__ void __launch_bounds__(256) spmm_coo_scale_kernel(const CooMmArgs<T> a, int c_row_major) {
    const int bi = blockIdx.z;
    if (a.flags && !a.flags[bi]) return;
    const T beta = a.s.b();
    T* C = a.C + bi * a.c_stride;
    const long long total = (long long)a.rows * a.n;
    for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (long long)gridDim.x * blockDim.x) {
        const long long i = c_row_major ? e / a.n : e % a.rows, j = c_row_major ? e % a.n : e / a.rows;
        T* p = C + i * a.sci + j * a.scj;
        *p = scaled(beta, p);
    }
}

// Atomic path, part 2: one atomic add of alpha * (run sum) per run of equal row index, lane and column.
template <typename T>
__global__ void __launch_bounds__(32 * COO_MM_WARPS) spmm_coo_atomic_kernel(const CooMmArgs<T> a) {
    const int lane = (int)threadIdx.x & 31;
    const int bi = blockIdx.z;
    if (a.flags && !a.flags[bi]) return;
    const int* row = a.row + bi * a.a_stride;
    const int* col = a.col + bi * a.a_stride;
    const T*   val = a.val + bi * a.a_stride;
    const T*   B = a.B + bi * a.b_stride;
    T*         C = a.C + bi * a.c_stride;
    const int panel = blockIdx.y;
    const int ja = panel * COO_MM_PANEL + lane, jb = ja + 32;
    const bool la = ja < a.n, lb = jb < a.n;
    const T alpha = a.s.a();
    auto add = [&](int r, T s0, T s1) {
        T* cr = C + (long long)r * a.sci;
        if (la) atomicAdd(cr + (long long)ja * a.scj, alpha * s0);
        if (lb) atomicAdd(cr + (long long)jb * a.scj, alpha * s1);
    };
    for (int chunk = blockIdx.x * COO_MM_WARPS + ((int)threadIdx.x >> 5); chunk < a.nchunks; chunk += gridDim.x * COO_MM_WARPS) {
        const int n0 = chunk * COO_MM_CHUNK, n1 = min(n0 + COO_MM_CHUNK, a.nnz);
        T acc0, acc1;
        const int last = walk_chunk(a, row, col, val, B, n0, n1, lane, ja, jb, la, lb, acc0, acc1,
                                    [&](int r, int, T s0, T s1) { add(r, s0, s1); });
        add(last, acc0, acc1);
    }
}

// Workspace layout: [flags: int per batch | carry rows: 2 ints per chunk and batch | carry values: 2 x 64 per chunk, panel and
// batch | row-major copy of B (one per batch matrix of B)].  SIZE_MAX when the size does not fit a size_t.
struct CooMmLayout {
    size_t flags = 0, carry_row = 0, carry_val = 0, bcopy = 0, total = 0;
    bool   copy_b = false;
};
static CooMmLayout coo_mm_layout(int dtype, int64_t kdim, int64_t n, int64_t nnz, int b_row_major, int batch, int64_t b_stride) {
    CooMmLayout l;
    const size_t vsz = dtype == 1 ? 8 : 4;
    const double nchunks = (double)((nnz + COO_MM_CHUNK - 1) / COO_MM_CHUNK), npanels = (double)((n + COO_MM_PANEL - 1) / COO_MM_PANEL);
    l.copy_b = !b_row_major && n >= COO_MM_MIN_N_FOR_TRANSPOSE && kdim > 0 && nnz > 0;
    const double nb = b_stride != 0 && batch > 1 ? batch : 1;
    const double est = 4.0 * batch + 8.0 * batch * nchunks + (double)vsz * batch * nchunks * npanels * 2 * COO_MM_PANEL +
                       (l.copy_b ? (double)vsz * nb * kdim * n : 0.0) + 1024.0;
    if (est > 9.0e18) { l.total = SIZE_MAX; return l; }
    const size_t nc = (size_t)nchunks, np = (size_t)npanels;
    l.flags = 0;
    l.carry_row = round_up_256((size_t)batch * 4);
    l.carry_val = l.carry_row + round_up_256((size_t)batch * nc * 2 * 4);
    l.bcopy = l.carry_val + round_up_256((size_t)batch * nc * np * 2 * COO_MM_PANEL * vsz);
    l.total = l.bcopy + (l.copy_b ? round_up_256((size_t)nb * (size_t)kdim * (size_t)n * vsz) : 0);
    return l;
}

template <typename T>
static int launch_coo_mm(cudaStream_t stream, int transpose, int64_t rows, int64_t cols, int64_t n, int64_t nnz, const void* row_ind,
                         const void* col_ind, const void* values, int base, const void* alpha, const void* beta, int on_device,
                         const void* B, int64_t ldb, int b_row_major, void* C, int64_t ldc, int c_row_major, int batch, int64_t a_stride,
                         int64_t b_stride, int64_t c_stride, void* ws, size_t ws_bytes) {
    const int dt = sizeof(T) == 8 ? 1 : 0;
    if (transpose) { std::swap(row_ind, col_ind); std::swap(rows, cols); }   // A^T: the same entries with the index arrays swapped
    if (batch == 1) a_stride = b_stride = c_stride = 0;
    const CooMmLayout l = coo_mm_layout(dt, cols, n, nnz, b_row_major, batch, b_stride);
    const bool ws_ok = l.total != SIZE_MAX && workspace_usable(ws, ws_bytes, l.total);
    const bool atomic_only = transpose || !ws_ok;
    CooMmArgs<T> a;
    a.row = (const int*)row_ind; a.col = (const int*)col_ind; a.val = (const T*)values; a.B = (const T*)B; a.C = (T*)C;
    a.base = base; a.rows = (int)rows; a.n = (int)n; a.nnz = (int)nnz;
    a.nchunks = (int)((nnz + COO_MM_CHUNK - 1) / COO_MM_CHUNK); a.npanels = (int)((n + COO_MM_PANEL - 1) / COO_MM_PANEL);
    a.a_stride = a_stride; a.b_stride = b_stride; a.c_stride = c_stride;
    if (ws_ok && l.copy_b) {                                          // the sample's layout: a row-major copy of each B in the buffer
        T* bt = (T*)((char*)ws + l.bcopy);
        const int cnt = b_stride != 0 ? batch : 1;
        for (int i = 0; i < cnt; i++) {
            const int rc = transpose_col_to_row_major(stream, dt, (const T*)B + (size_t)i * b_stride, ldb, bt + (size_t)i * cols * n, cols, n);
            if (rc != 0) return rc;
        }
        a.B = bt; b_row_major = 1; ldb = n; a.b_stride = b_stride != 0 ? cols * n : 0;
    }
    a.sbk = b_row_major ? ldb : 1; a.sbj = b_row_major ? 1 : ldb;
    a.sci = c_row_major ? ldc : 1; a.scj = c_row_major ? 1 : ldc;
    set_scalars(a.s, alpha, beta, on_device);
    a.flags = nullptr; a.carry_row = nullptr; a.carry_val = nullptr;
    const long long cells = rows * n;
    const dim3 sgrid((unsigned)std::max<long long>(1, std::min<long long>((cells + 255) / 256, COO_MM_STRIDE_CTAS)), 1, (unsigned)batch);
    if (nnz == 0) {                                                   // C = beta * C
        spmm_coo_scale_kernel<T><<<sgrid, 256, 0, stream>>>(a, c_row_major);
        return (int)cudaGetLastError();
    }
    if (!atomic_only) {
        int* flags = (int*)((char*)ws + l.flags);
        cudaError_t e = cudaMemsetAsync(flags, 0, (size_t)batch * sizeof(int), stream);
        if (e != cudaSuccess) return (int)e;
        a.flags = flags; a.carry_row = (int*)((char*)ws + l.carry_row); a.carry_val = (T*)((char*)ws + l.carry_val);
        const dim3 cgrid((unsigned)std::max<long long>(1, std::min<long long>((nnz + 255) / 256, COO_MM_STRIDE_CTAS)), 1, (unsigned)batch);
        spmm_coo_check_kernel<<<cgrid, 256, 0, stream>>>(a.row, a.nnz, a.a_stride, flags);
        const dim3 grid((unsigned)((a.nchunks + COO_MM_WARPS - 1) / COO_MM_WARPS), (unsigned)a.npanels, (unsigned)batch);
        spmm_coo_sorted_kernel<T><<<grid, 32 * COO_MM_WARPS, 0, stream>>>(a);
        const dim3 fgrid((unsigned)((2 * a.nchunks + COO_MM_WARPS - 1) / COO_MM_WARPS), (unsigned)a.npanels, (unsigned)batch);
        spmm_coo_fixup_kernel<T><<<fgrid, 32 * COO_MM_WARPS, 0, stream>>>(a);
    }
    spmm_coo_scale_kernel<T><<<sgrid, 256, 0, stream>>>(a, c_row_major);
    const dim3 agrid((unsigned)std::min<long long>((a.nchunks + COO_MM_WARPS - 1) / COO_MM_WARPS, COO_MM_STRIDE_CTAS), (unsigned)a.npanels,
                     (unsigned)batch);
    spmm_coo_atomic_kernel<T><<<agrid, 32 * COO_MM_WARPS, 0, stream>>>(a);
    return (int)cudaGetLastError();
}

}  // namespace b200

using namespace b200;

extern "C" {

void b200spmm_coo_params(int32_t* chunk_nnz, int32_t* panel_cols, int64_t* flag_offset) {
    if (chunk_nnz) *chunk_nnz = COO_MM_CHUNK;
    if (panel_cols) *panel_cols = COO_MM_PANEL;
    if (flag_offset) *flag_offset = 0;
}

size_t b200spmm_coo_workspace_bytes(int dtype, int transpose_a, int64_t rows, int64_t cols, int64_t n, int64_t nnz, int b_row_major,
                                    int batch, int64_t b_stride) {
    if ((dtype != 0 && dtype != 1) || rows < 0 || cols < 0 || n < 0 || nnz < 0 || batch < 1) return 0;
    return coo_mm_layout(dtype, transpose_a ? rows : cols, n, nnz, b_row_major, batch, b_stride).total;
}

int b200spmm_coo(void* stream, int dtype, int transpose_a, int64_t rows, int64_t cols, int64_t n, int64_t nnz, const void* row_ind,
                 const void* col_ind, const void* values, int32_t base, const void* alpha, const void* beta, int scalars_on_device,
                 const void* B, int64_t ldb, int b_row_major, void* C, int64_t ldc, int c_row_major, int batch, int64_t a_stride,
                 int64_t b_stride, int64_t c_stride, void* workspace, size_t workspace_bytes) {
    if (dtype != 0 && dtype != 1) return -1;
    if (rows < 0 || cols < 0 || n < 0 || nnz < 0 || !alpha || !beta || (base != 0 && base != 1)) return -1;
    if (batch < 1 || batch > 65535 || a_stride < 0 || b_stride < 0 || c_stride < 0) return -1;
    if (rows > INT32_MAX - 64 || cols > INT32_MAX - 64 || n > INT32_MAX - 64 || nnz > INT32_MAX - 65536) return -1;
    if ((n + COO_MM_PANEL - 1) / COO_MM_PANEL > 65535) return -1;
    const int64_t crows = transpose_a ? cols : rows, kdim = transpose_a ? rows : cols;      // C is crows x n, B kdim x n
    if (ldb < (b_row_major ? n : kdim) || ldc < (c_row_major ? n : crows) || ldb < 1 || ldc < 1) return -1;
    if (batch > 1 && c_stride < (c_row_major ? crows : n) * ldc) return -1;                 // the batch's outputs would overlap
    if (crows == 0 && nnz > 0) return -1;
    if (crows == 0 || n == 0) return 0;
    if (!C || (nnz > 0 && (!row_ind || !col_ind || !values || !B))) return -1;
    if (dtype == 0)
        return launch_coo_mm<float>((cudaStream_t)stream, transpose_a, rows, cols, n, nnz, row_ind, col_ind, values, base, alpha, beta,
                                    scalars_on_device, B, ldb, b_row_major, C, ldc, c_row_major, batch, a_stride, b_stride, c_stride,
                                    workspace, workspace_bytes);
    return launch_coo_mm<double>((cudaStream_t)stream, transpose_a, rows, cols, n, nnz, row_ind, col_ind, values, base, alpha, beta,
                                 scalars_on_device, B, ldb, b_row_major, C, ldc, c_row_major, batch, a_stride, b_stride, c_stride,
                                 workspace, workspace_bytes);
}

}  // extern "C"
