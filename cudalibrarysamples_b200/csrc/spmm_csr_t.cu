// spmm_csr_t.cu -- transposed CSR x dense  C = alpha * A^T * op(B) + beta * C  on H100 (sm_90a), A rows x cols CSR with int32
// offsets / columns (base 0 or 1): fp32 / fp64, and fp16 / bf16 with fp32 compute.  The backward pass of a graph layer (A^T * G on
// the pattern whose forward pass is A * X), the normal equations, any two-sided operator.  For real types opA = C is opA = T.
//
// No atomics: A^T is materialised once as a CSR matrix of its own (a "transposed plan", the CSC form of A) and every call runs the
// existing opA = N kernels on it -- spmm_csr_kernel / spmm_csr_ctile_kernel (spmm_csr.cu) for fp32 / fp64, spmm_csr16_kernel and
// its carry fix-up (spmm_csr16.cu) for fp16 / bf16.  The result is deterministic, and bit-identical to an opA = N call on the
// explicit transpose.
//
// The plan, from the pattern alone (row offsets and columns):
//   tOff[cols + 1]  CSC column pointers (base 0);
//   tRow[nnz]       the row of each CSC entry (base 0);
//   perm[nnz]       the CSR position of each CSC entry.
// Within a column, entries are in ascending row order (that of scipy.sparse.csr_matrix.tocsc()), so the plan is a pure function of
// the pattern.  It is a stable LSD radix sort of the entry indices by column (radix_sort.cuh, shared with convert.cu), 8 bits per
// pass (as many passes as cols - 1 needs bits, at least one): per tile of RT_TILE entries a digit histogram, a scan of the histograms
// per digit, then a scatter that ranks the entries of a tile in their CSR order.  Stable ranking keeps equal columns in entry order, and entry order is row order.  The
// sorted keys give tOff, a binary search over the row offsets gives tRow.  Each call then gathers tVal[k] = val[perm[k]], so new
// values (cusparseSpMatSetValues) need no new plan; a new pattern does.
//
// Workspace (the caller's, 16-byte aligned; every part 256-byte aligned, b200spmm_csr_t_layout):
//   [ plan: tOff | tRow | perm ][ sort scratch: keys x2 | indices x2 | histograms | digit totals ][ tVal ][ the N kernel's workspace ]
// The plan and the scratch depend on (cols, nnz) only.  No allocation, no host synchronisation: graph-capturable.
#include "spmv_common.cuh"
#include "radix_sort.cuh"
#include "../../include/b200spmv.h"

#include <algorithm>
#include <cub/block/block_scan.cuh>

namespace b200 {

constexpr int RT_WARPS = RT_THREADS / 32;
constexpr int T_F32 = 0, T_F64 = 1, T_F16 = 2, T_BF16 = 14;   // cudaDataType values

static_assert(RT_BINS == RT_THREADS, "one thread per digit");

// key of entry i: keys[i], or keys[kidx[i]] when the keys are read through an earlier permutation, less sub (a base)
__device__ __forceinline__ int rt_key(const int* keys, int sub, const int* kidx, int i) {
    return __ldg(keys + (kidx ? __ldg(kidx + i) : i)) - sub;
}

// hist[d * ntiles + t] = entries of tile t whose digit is d
__global__ void __launch_bounds__(RT_THREADS) spmm_csr_t_hist_kernel(const int* keys, int sub, const int* kidx, int nnz, int shift,
                                                                  int* hist, int ntiles) {
    __shared__ int h[RT_BINS];
    h[threadIdx.x] = 0;
    __syncthreads();
    const int t0 = (int)blockIdx.x * RT_TILE;
#pragma unroll
    for (int r = 0; r < RT_ITEMS; r++) {
        const int i = t0 + r * RT_THREADS + (int)threadIdx.x;
        if (i < nnz) atomicAdd(&h[(rt_key(keys, sub, kidx, i) >> shift) & (RT_BINS - 1)], 1);
    }
    __syncthreads();
    hist[(long long)threadIdx.x * ntiles + blockIdx.x] = h[threadIdx.x];
}

// One CTA per digit d: hist[d * ntiles + t] becomes the entries of digit d in tiles before t; tot[d] the digit's total.
__global__ void __launch_bounds__(RT_THREADS) spmm_csr_t_scan_kernel(int* hist, int ntiles, int* tot) {
    using Scan = cub::BlockScan<int, RT_THREADS>;
    __shared__ typename Scan::TempStorage tmp;
    int* row = hist + (long long)blockIdx.x * ntiles;
    int carry = 0;
    for (int t0 = 0; t0 < ntiles; t0 += RT_THREADS) {
        const int t = t0 + (int)threadIdx.x;
        const int v = t < ntiles ? row[t] : 0;
        int ex, sum;
        Scan(tmp).ExclusiveSum(v, ex, sum);
        if (t < ntiles) row[t] = carry + ex;
        carry += sum;
        __syncthreads();                               // tmp is reused
    }
    if (threadIdx.x == 0) tot[blockIdx.x] = carry;
}

// Stable scatter of one tile: entry i goes to (entries of smaller digits) + (entries of its digit in earlier tiles) + (entries of its
// digit before it in this tile).  Within a round of RT_THREADS entries, warps in order and lanes in order; rounds in order.
// vals == nullptr: the indices are the entry positions themselves (the first pass).
__global__ void __launch_bounds__(RT_THREADS) spmm_csr_t_scatter_kernel(const int* keys, int sub, const int* kidx, const int* vals, int nnz,
                                                                     int shift, const int* hist, const int* tot, int ntiles,
                                                                     int* keys_out, int* vals_out) {
    using Scan = cub::BlockScan<int, RT_THREADS>;
    __shared__ typename Scan::TempStorage tmp;
    __shared__ int base[RT_BINS];                      // next position of each digit
    __shared__ int wc[RT_WARPS][RT_BINS];              // per round: entries of digit d in warps before w (after the scan)
    const int tid = (int)threadIdx.x, lane = tid & 31, warp = tid >> 5;
    int digit_base;
    Scan(tmp).ExclusiveSum(__ldg(tot + tid), digit_base);
    base[tid] = digit_base + __ldg(hist + (long long)tid * ntiles + blockIdx.x);
#pragma unroll
    for (int w = 0; w < RT_WARPS; w++) wc[w][tid] = 0;
    __syncthreads();
    const unsigned lt = (1u << lane) - 1u;
    const int t0 = (int)blockIdx.x * RT_TILE;
#pragma unroll 1
    for (int r = 0; r < RT_ITEMS; r++) {
        const int i = t0 + r * RT_THREADS + tid;
        const bool live = i < nnz;
        const int key = live ? rt_key(keys, sub, kidx, i) : 0;
        const int d = live ? (key >> shift) & (RT_BINS - 1) : -1;
        const unsigned peers = __match_any_sync(0xffffffffu, d);
        const int rank = __popc(peers & lt);
        if (live && rank == 0) wc[warp][d] = __popc(peers);
        __syncthreads();
        int s = 0;
#pragma unroll
        for (int w = 0; w < RT_WARPS; w++) { const int c = wc[w][tid]; wc[w][tid] = s; s += c; }
        __syncthreads();
        if (live) {
            const int pos = base[d] + wc[warp][d] + rank;
            keys_out[pos] = key;
            vals_out[pos] = vals ? __ldg(vals + i) : i;
        }
        __syncthreads();
        base[tid] += s;
#pragma unroll
        for (int w = 0; w < RT_WARPS; w++) wc[w][tid] = 0;
        __syncthreads();
    }
}

// Offsets from sorted keys (less sub): entry k is the first of every key in (key[k - 1], key[k]]; k = nnz closes the keys up to
// nkeys.  Clamped to [0, nkeys]: keys from a caller's array may hold anything.
__global__ void __launch_bounds__(RT_THREADS) spmm_csr_t_offsets_kernel(const int* sorted, int sub, int nnz, int nkeys, int base,
                                                                     int* t_off) {
    for (long long k = (long long)blockIdx.x * RT_THREADS + threadIdx.x; k <= nnz; k += (long long)gridDim.x * RT_THREADS) {
        const long long prev = k > 0 ? (long long)sorted[k - 1] - sub : -1, cur = k < nnz ? (long long)sorted[k] - sub : nkeys;
        const long long hi = cur < nkeys ? cur : nkeys;
        for (long long c = prev + 1 > 0 ? prev + 1 : 0; c <= hi; c++) t_off[c] = (int)k + base;
    }
}

// tRow[k] = out_base + the row holding CSR entry perm[k] (entry k when perm is NULL): the last r with off[r] - base <= perm[k]
__global__ void __launch_bounds__(RT_THREADS) spmm_csr_t_rows_kernel(const int* off, int base, int rows, const int* perm, int nnz,
                                                                  int out_base, int* t_row) {
    const int k = (int)blockIdx.x * RT_THREADS + (int)threadIdx.x;
    if (k >= nnz) return;
    t_row[k] = csr_row_of(off, rows, base, perm ? perm[k] : k) + out_base;
}

// tVal[k] = val[perm[k]], bit for bit (W: the value's width as an unsigned type)
template <typename W>
__global__ void __launch_bounds__(RT_THREADS) spmm_csr_t_gather_kernel(const W* val, const int* perm, int nnz, W* t_val) {
    const int k = (int)blockIdx.x * RT_THREADS + (int)threadIdx.x;
    if (k < nnz) t_val[k] = __ldg(val + ldg_stream(perm + k));
}

// ------------------------------------------------------------------------------------------------ host side
static int64_t rt_ntiles(int64_t nnz) { return (nnz + RT_TILE - 1) / RT_TILE; }
static unsigned rt_grid(int64_t n) { return (unsigned)((n + RT_THREADS - 1) / RT_THREADS); }

int rt_passes(int64_t nkeys) {
    int bits = 0;
    while (bits < 32 && ((int64_t)1 << bits) < nkeys) bits++;   // bits of nkeys - 1
    return bits == 0 ? 1 : (bits + RT_BITS - 1) / RT_BITS;
}

size_t rt_scratch_bytes(int64_t n) {
    return 4 * round_up_256((size_t)n * 4) + round_up_256((size_t)RT_BINS * rt_ntiles(n) * 4) + round_up_256((size_t)RT_BINS * 4);
}

RtScratch rt_scratch(char* base, int64_t n) {
    const size_t e = round_up_256((size_t)n * 4);
    RtScratch s;
    s.k[0] = (int*)base;
    s.k[1] = (int*)(base + e);
    s.v[0] = (int*)(base + 2 * e);
    s.v[1] = (int*)(base + 3 * e);
    s.hist = (int*)(base + 4 * e);
    s.tot = (int*)(base + 4 * e + round_up_256((size_t)RT_BINS * rt_ntiles(n) * 4));
    return s;
}

void rt_sort(cudaStream_t st, const int* keys, int sub, const int* kidx, const int* vals, int n, int64_t nkeys, const RtScratch& s,
             int* vals_out, const int** sorted_keys, const int** sorted_vals) {
    const int ntiles = (int)rt_ntiles(n), passes = rt_passes(nkeys);
    for (int p = 0; p < passes; p++) {
        const int shift = p * RT_BITS;
        int* ko = s.k[p & 1];
        int* vo = p == passes - 1 && vals_out ? vals_out : s.v[p & 1];
        spmm_csr_t_hist_kernel<<<ntiles, RT_THREADS, 0, st>>>(keys, sub, kidx, n, shift, s.hist, ntiles);
        spmm_csr_t_scan_kernel<<<RT_BINS, RT_THREADS, 0, st>>>(s.hist, ntiles, s.tot);
        spmm_csr_t_scatter_kernel<<<ntiles, RT_THREADS, 0, st>>>(keys, sub, kidx, vals, n, shift, s.hist, s.tot, ntiles, ko, vo);
        keys = ko; vals = vo; kidx = nullptr; sub = 0;
    }
    if (sorted_keys) *sorted_keys = keys;
    if (sorted_vals) *sorted_vals = vals;
}

void rt_offsets(cudaStream_t st, const int* keys, int sub, int n, int64_t nkeys, int base, int* out) {
    const unsigned grid = (unsigned)std::min<long long>(rt_grid((int64_t)n + 1), 65536);
    spmm_csr_t_offsets_kernel<<<grid, RT_THREADS, 0, st>>>(keys, sub, n, (int)nkeys, base, out);
}

void rt_rows(cudaStream_t st, const int* off, int off_base, int64_t rows, const int* perm, int n, int out_base, int* out) {
    spmm_csr_t_rows_kernel<<<rt_grid(n), RT_THREADS, 0, st>>>(off, off_base, (int)rows, perm, n, out_base, out);
}

bool rt_gather(cudaStream_t st, int width, const void* src, const int* perm, int n, void* dst) {
    const unsigned g = rt_grid(n);
    switch (width) {
    case 1: spmm_csr_t_gather_kernel<unsigned char><<<g, RT_THREADS, 0, st>>>((const unsigned char*)src, perm, n, (unsigned char*)dst); break;
    case 2: spmm_csr_t_gather_kernel<unsigned short><<<g, RT_THREADS, 0, st>>>((const unsigned short*)src, perm, n, (unsigned short*)dst); break;
    case 4: spmm_csr_t_gather_kernel<unsigned><<<g, RT_THREADS, 0, st>>>((const unsigned*)src, perm, n, (unsigned*)dst); break;
    case 8: spmm_csr_t_gather_kernel<unsigned long long><<<g, RT_THREADS, 0, st>>>((const unsigned long long*)src, perm, n, (unsigned long long*)dst); break;
    case 16: spmm_csr_t_gather_kernel<uint4><<<g, RT_THREADS, 0, st>>>((const uint4*)src, perm, n, (uint4*)dst); break;
    default: return false;
    }
    return true;
}

static size_t elem_bytes(int dtype) { return dtype == T_F64 ? 8 : dtype == T_F32 ? 4 : 2; }
static bool is16(int dtype) { return dtype == T_F16 || dtype == T_BF16; }

struct TLayout {
    size_t t_off, t_row, perm, k0, t_val, ws, ws_bytes, total;
};

static TLayout t_layout(int dtype, int64_t rows, int64_t cols, int64_t n, int64_t nnz, int64_t sbk, int64_t sbj) {
    TLayout L;
    const size_t e = (size_t)nnz * 4;
    L.t_off = 0;
    L.t_row = round_up_256(((size_t)cols + 1) * 4);
    L.perm = L.t_row + round_up_256(e);
    L.k0 = L.perm + round_up_256(e);
    L.t_val = L.k0 + rt_scratch_bytes(nnz);
    L.ws = L.t_val + round_up_256((size_t)nnz * elem_bytes(dtype));
    // the N kernel's workspace for the cols x rows CSR matrix A^T: the row-major copy of a K-contiguous B (and the 16-bit carry slots)
    if (is16(dtype)) L.ws_bytes = b200spmm_csr16_workspace_bytes(rows, n, nnz, sbk, sbj);
    else L.ws_bytes = b200spmm_csr_workspace_bytes(dtype, rows, n, sbj == 1 ? 1 : 0);
    L.total = L.ws + round_up_256(L.ws_bytes);
    return L;
}

static bool dims_ok(int64_t rows, int64_t cols, int64_t nnz) {
    return rows >= 0 && cols >= 0 && nnz >= 0 && rows <= INT32_MAX - 64 && cols <= INT32_MAX - 64 && nnz <= INT32_MAX - 65536 &&
           (nnz == 0 || (rows > 0 && (nnz + rows - 1) / rows <= cols));
}

static int build_plan(cudaStream_t st, int64_t rows, int64_t cols, int64_t nnz, const int* off, const int* col, int base, char* ws) {
    const TLayout L = t_layout(T_F32, rows, cols, 0, nnz, 0, 0);
    int* t_off = (int*)(ws + L.t_off);
    int* perm = (int*)(ws + L.perm);
    const int nz = (int)nnz;
    if (nz > 0) {
        const int* sorted = nullptr;
        rt_sort(st, col, base, nullptr, nullptr, nz, cols, rt_scratch(ws + L.k0, nnz), perm, &sorted, nullptr);
        rt_offsets(st, sorted, 0, nz, cols, 0, t_off);
        rt_rows(st, off, base, rows, perm, nz, 0, (int*)(ws + L.t_row));
    } else {
        rt_offsets(st, nullptr, 0, 0, cols, 0, t_off);
    }
    return (int)cudaGetLastError();
}

}  // namespace b200

using namespace b200;

extern "C" {

size_t b200spmm_csr_t_layout(int dtype, int64_t rows, int64_t cols, int64_t n, int64_t nnz, int64_t sbk, int64_t sbj, size_t* offsets) {
    if (!dims_ok(rows, cols, nnz) || n < 0 || sbk < 0 || sbj < 0) return 0;
    if (dtype != T_F32 && dtype != T_F64 && !is16(dtype)) return 0;
    const TLayout L = t_layout(dtype, rows, cols, n, nnz, sbk, sbj);
    if (offsets) {
        offsets[0] = L.t_off; offsets[1] = L.t_row; offsets[2] = L.perm; offsets[3] = L.k0; offsets[4] = L.t_val; offsets[5] = L.ws;
    }
    return L.total;
}

size_t b200spmm_csr_t_workspace_bytes(int dtype, int64_t rows, int64_t cols, int64_t n, int64_t nnz, int64_t sbk, int64_t sbj) {
    return b200spmm_csr_t_layout(dtype, rows, cols, n, nnz, sbk, sbj, nullptr);
}

int b200spmm_csr_t_plan(void* stream, int64_t rows, int64_t cols, int64_t nnz, const void* offsets, const void* columns, int32_t base,
                        void* workspace, size_t workspace_bytes) {
    if (!dims_ok(rows, cols, nnz) || (base != 0 && base != 1)) return -1;
    if (!offsets || (nnz > 0 && !columns) || !workspace || ((uintptr_t)workspace & 15)) return -1;
    if (workspace_bytes < t_layout(T_F32, rows, cols, 0, nnz, 0, 0).t_val) return -1;
    return build_plan((cudaStream_t)stream, rows, cols, nnz, (const int*)offsets, (const int*)columns, base, (char*)workspace);
}

int b200spmm_csr_t(void* stream, int dtype, int c_type, int64_t rows, int64_t cols, int64_t n, int64_t nnz, const void* offsets,
                   const void* columns, const void* values, int32_t base, const void* alpha, const void* beta, int scalars_on_device,
                   const void* B, int64_t sbk, int64_t sbj, void* C, int64_t ldc, int c_row_major, int plan_valid, void* workspace,
                   size_t workspace_bytes) {
    // every check of the N entry point (for the cols x rows matrix A^T) is made here, before anything is launched
    const bool h16 = is16(dtype);
    if (dtype != T_F32 && dtype != T_F64 && !h16) return -1;
    if (h16 ? (c_type != dtype && c_type != T_F32) : c_type != dtype) return -1;
    if (!dims_ok(rows, cols, nnz) || n < 0 || !alpha || !beta || (base != 0 && base != 1) || sbk < 0 || sbj < 0) return -1;
    if (h16 ? n > 32 * 65535 : (n > INT32_MAX - 64 || (n + 63) / 64 > 65535)) return -1;
    if (ldc < 1 || ldc < (c_row_major ? n : cols)) return -1;
    int b_row_major = 1;
    int64_t ldb = sbk;
    if (!h16) {                                        // fp32 / fp64: op(B) row-major (sbj == 1) or column-major (sbk == 1)
        if (sbj != 1) { if (sbk != 1) return -1; b_row_major = 0; ldb = sbj; }
        if (ldb < (b_row_major ? n : rows)) return -1;
    }
    if (cols == 0 || n == 0) return 0;
    if (!C || !offsets || (nnz > 0 && (!columns || !values || !B))) return -1;
    if (!workspace || ((uintptr_t)workspace & 15)) return -1;
    const TLayout L = t_layout(dtype, rows, cols, n, nnz, sbk, sbj);
    if (workspace_bytes < L.total) return -1;
    const cudaStream_t st = (cudaStream_t)stream;
    char* ws = (char*)workspace;
    if (!plan_valid) {
        const int rc = build_plan(st, rows, cols, nnz, (const int*)offsets, (const int*)columns, base, ws);
        if (rc != 0) return rc;
    }
    const int* t_off = (const int*)(ws + L.t_off);
    const int* t_row = (const int*)(ws + L.t_row);
    const int* perm = (const int*)(ws + L.perm);
    void* t_val = ws + L.t_val;
    if (nnz > 0) {
        rt_gather(st, (int)elem_bytes(dtype), values, perm, (int)nnz, t_val);
        const cudaError_t e = cudaGetLastError();
        if (e != cudaSuccess) return (int)e;
    }
    if (h16)
        return b200spmm_csr16(stream, dtype, c_type, cols, rows, n, nnz, t_off, t_row, t_val, 0, alpha, beta, scalars_on_device, B, sbk,
                              sbj, C, ldc, c_row_major, ws + L.ws, L.ws_bytes);
    return b200spmm_csr_ws(stream, dtype, cols, rows, n, nnz, t_off, t_row, t_val, 0, alpha, beta, scalars_on_device, B, ldb, b_row_major,
                           C, ldc, c_row_major, L.ws_bytes ? ws + L.ws : nullptr);
}

}  // extern "C"
