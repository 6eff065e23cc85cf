// dense_convert.cu -- sparse <-> dense conversion on H100 (sm_90a), int32 indices: CSR / CSC / COO / Blocked-ELL -> dense
// (cusparseSparseToDense) and dense -> CSR / CSC / Blocked-ELL (cusparseDenseToSparse_convert).  DESIGN.md 3.24.
//
// Values move by width (2, 4, 8 or 16 bytes), never through arithmetic, so every fp16 ... complex128 value keeps its bits, NaN
// payloads included; no floating-point atomics, so every result is a pure function of the input -- except COO -> dense with
// duplicate (row, col) pairs, where one thread per entry stores and which of the duplicates' values lands is unspecified.  No
// allocation, no host synchronisation: graph-capturable.
//
// CSC of A is CSR of A^T, and a row-major A is a column-major A^T, so CSR and CSC share two kernel shapes over a "major" index i
// (the CSR row / CSC column) and a "minor" index j:
//   along   the dense contiguous dimension is the minor one (CSR <-> row-major, CSC <-> column-major): element (i, j) at i * ld + j.
//           One warp per major line.
//   across  the dense contiguous dimension is the major one (CSR <-> column-major, CSC <-> row-major): element (i, j) at i + j * ld.
//           A CTA per panel of 32 major lines, so every dense access covers 32 consecutive elements.
// Sparse -> dense writes every element of the window once as zero, then scatters the entries, in the same warp / CTA (ordered by
// __syncwarp / __syncthreads) so the scatter lands in lines still in L2.  Within a major line, entries scatter in storage order,
// 32 at a time, and of equal minor indices in one chunk only the last stores (__match_any_sync): the last duplicate wins.  Nothing
// outside the window is written: not the ld padding, not an entry whose index lies outside the matrix.
// Dense -> sparse writes entry k of line i at off[i] + k (base removed) in ascending minor order, counted by __ballot_sync /
// __popc, and never outside [off[i], off[i + 1]): a line with more non-zeros than its offsets allow keeps the first ones, one with
// fewer leaves the rest of its range unwritten.  The non-zero predicate is the closed analysis's, pinned on the H100 (DESIGN.md
// 3.24): "v != 0" per part without flushing denormals (+-0 are zero; denormals, Inf and NaN are not), except that a 16-bit value
// whose magnitude bits exceed 0x7C00 is zero; a complex value is non-zero when either part is.
#include <cuda_runtime.h>

#include <cstdint>

#include "../../include/b200spmv.h"

namespace b200 {

constexpr int DC_THREADS = 256;      // along kernels and the COO / Blocked-ELL kernels
constexpr int DC_PANEL = 32;         // major lines per CTA of the across kernels
constexpr int DC_MAPW = 4096;        // block columns per shared-memory window of bell2dense
constexpr int ORDER_COL = 1, ORDER_ROW = 2;   // cusparseOrder_t
// dense -> Blocked-ELL writes zeros into the slots of the -1 padding, as the closed library's convert does (DESIGN.md 3.24)
constexpr int DC_BELL_PAD_ZERO = 1;

template <int W> struct Bits;
template <> struct Bits<2> { using T = unsigned short; };
template <> struct Bits<4> { using T = unsigned int; };
template <> struct Bits<8> { using T = uint2; };
template <> struct Bits<16> { using T = uint4; };

template <typename V> __device__ __forceinline__ V zero_value() { V v; memset(&v, 0, sizeof(V)); return v; }

// "v != 0" as the closed library's analysis counts it, per part of pw bytes (pw = the width, or half of it for a complex type):
// any magnitude bit set, so denormals, Inf and NaN count and +-0 do not -- except a 16-bit value, whose bits that analysis reads
// as fp16 whatever the type: magnitude bits above 0x7C00 (an fp16 NaN; for bf16 every value from about 2.7e36 up, Inf and NaN) are
// zero.  Pinned over all 65536 patterns of each 16-bit type on the H100 (DESIGN.md 3.24).  Whole words, so nothing leaves registers.
__device__ __forceinline__ bool nonzero(unsigned short v, int) {
    const unsigned mag = v & 0x7FFFu;
    return mag != 0 && mag <= 0x7C00u;
}
__device__ __forceinline__ bool nonzero(unsigned v, int) { return (v & 0x7FFFFFFFu) != 0; }
__device__ __forceinline__ bool nonzero(uint2 v, int pw) {          // fp64 (pw 8) or complex fp32 (pw 4); little-endian
    return pw == 8 ? (v.x | (v.y & 0x7FFFFFFFu)) != 0 : ((v.x | v.y) & 0x7FFFFFFFu) != 0;
}
__device__ __forceinline__ bool nonzero(uint4 v, int) { return (v.x | (v.y & 0x7FFFFFFFu) | v.z | (v.w & 0x7FFFFFFFu)) != 0; }

// element k of a 16-byte vector of 16 / sizeof(V) elements; k a compile-time constant after unrolling
__device__ __forceinline__ unsigned word(const uint4& u, int i) { return i == 0 ? u.x : i == 1 ? u.y : i == 2 ? u.z : u.w; }
template <typename V> __device__ __forceinline__ V element(const uint4& u, int k);
template <> __device__ __forceinline__ unsigned short element(const uint4& u, int k) {
    return (unsigned short)(word(u, k >> 1) >> ((k & 1) * 16));
}
template <> __device__ __forceinline__ unsigned element(const uint4& u, int k) { return word(u, k); }
template <> __device__ __forceinline__ uint2 element(const uint4& u, int k) { return make_uint2(word(u, 2 * k), word(u, 2 * k + 1)); }
template <> __device__ __forceinline__ uint4 element(const uint4& u, int) { return u; }

// zero the n elements at p, 16-byte stores on the aligned interior, scalar head and tail; lanes `lane` of `lanes`
template <typename V>
__device__ __forceinline__ void zero_line(V* p, long long n, int lane, int lanes) {
    constexpr int K = 16 / (int)sizeof(V);
    const long long mis = (long long)(((uintptr_t)p & 15) / sizeof(V));
    const long long head = mis ? (long long)K - mis < n ? (long long)K - mis : n : 0;
    const V z = zero_value<V>();
    for (long long j = lane; j < head; j += lanes) p[j] = z;
    const long long nv = (n - head) / K;
    uint4* q = (uint4*)(p + head);
    for (long long v = lane; v < nv; v += lanes) q[v] = make_uint4(0, 0, 0, 0);
    for (long long j = head + nv * K + lane; j < n; j += lanes) p[j] = z;
}

// scatter the entries [beg, end) of one major line, 32 at a time in storage order; of equal minor indices in a chunk the last
// stores, and chunks are ordered by __syncwarp: the last duplicate in storage order wins.  Whole warp, converged.
template <typename V>
__device__ __forceinline__ void scatter_line(V* dense, long long i, long long ld, bool along, long long nminor, const int* ind,
                                             const V* val, long long beg, long long end, int base, int lane) {
    for (long long e0 = beg; e0 < end; e0 += 32) {
        const long long e = e0 + lane;
        const bool act = e < end;
        const int j = act ? __ldg(ind + e) - base : -1;
        V v;
        if (act) v = val[e];
        const unsigned grp = __match_any_sync(0xffffffffu, j);
        const bool last = (grp >> lane) == 1u;
        if (act && last && j >= 0 && j < nminor) dense[along ? i * ld + j : i + (long long)j * ld] = v;
        __syncwarp();
    }
}

// offset k of a line with the base removed, clamped to [0, nnz]: no entry outside the arrays is ever touched
__device__ __forceinline__ long long entry(const int* off, long long k, int base, long long nnz) {
    const long long e = (long long)__ldg(off + k) - base;
    return e < 0 ? 0 : e > nnz ? nnz : e;
}

template <typename V>
__global__ void __launch_bounds__(DC_THREADS) csr2dense_along_kernel(long long M, long long N, long long nnz, const int* off, const int* ind,
                                                                     const V* val, int base, V* dense, long long ld) {
    const int lane = threadIdx.x & 31;
    const long long warps = (long long)gridDim.x * (DC_THREADS / 32);
    for (long long i = (long long)blockIdx.x * (DC_THREADS / 32) + (threadIdx.x >> 5); i < M; i += warps) {
        zero_line(dense + i * ld, N, lane, 32);
        __syncwarp();
        scatter_line(dense, i, ld, true, N, ind, val, entry(off, i, base, nnz), entry(off, i + 1, base, nnz), base, lane);
    }
}

template <typename V>
__global__ void __launch_bounds__(DC_THREADS) csr2dense_across_kernel(long long M, long long N, long long nnz, const int* off, const int* ind,
                                                                      const V* val, int base, V* dense, long long ld) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const V z = zero_value<V>();
    for (long long i0 = (long long)blockIdx.x * DC_PANEL; i0 < M; i0 += (long long)gridDim.x * DC_PANEL) {
        const int pr = M - i0 < DC_PANEL ? (int)(M - i0) : DC_PANEL;
        for (long long t = threadIdx.x; t < N * DC_PANEL; t += DC_THREADS) {
            const int r = (int)(t % DC_PANEL);
            if (r < pr) dense[i0 + r + (t / DC_PANEL) * ld] = z;
        }
        __syncthreads();
        for (int r = warp; r < pr; r += DC_THREADS / 32)
            scatter_line(dense, i0 + r, ld, false, N, ind, val, entry(off, i0 + r, base, nnz), entry(off, i0 + r + 1, base, nnz), base,
                         lane);
        __syncthreads();
    }
}

// zero the rows x cols window: one warp per dense line (a row of a row-major matrix, a column of a column-major one)
template <typename V>
__global__ void __launch_bounds__(DC_THREADS) zero_window_kernel(long long lines, long long len, V* dense, long long ld) {
    const long long warps = (long long)gridDim.x * (DC_THREADS / 32);
    for (long long l = (long long)blockIdx.x * (DC_THREADS / 32) + (threadIdx.x >> 5); l < lines; l += warps)
        zero_line(dense + l * ld, len, threadIdx.x & 31, 32);
}

// COO entries scattered into the zeroed window, one thread per entry; entries outside the matrix are skipped
template <typename V>
__global__ void __launch_bounds__(DC_THREADS) coo_scatter_kernel(long long m, long long n, long long nnz, const int* rows,
                                                                 const int* cols, const V* val, int base, V* dense, long long ld,
                                                                 int row_major) {
    for (long long e = (long long)blockIdx.x * DC_THREADS + threadIdx.x; e < nnz; e += (long long)gridDim.x * DC_THREADS) {
        const long long r = (long long)__ldg(rows + e) - base, c = (long long)__ldg(cols + e) - base;
        if (r >= 0 && r < m && c >= 0 && c < n) dense[row_major ? r * ld + c : r + c * ld] = val[e];
    }
}

// Blocked-ELL -> dense, one CTA per block row: a shared map from block column to the last slot naming it (integer atomicMax, so
// the last duplicate slot wins), then every element of the block row's window written once, from its slot or as zero.  Slots
// whose column lies outside the matrix (the -1 padding among them) are never read.
template <typename V>
__global__ void __launch_bounds__(DC_THREADS) bell2dense_kernel(long long m, long long n, int bs, int eb, const int* colind,
                                                                const V* val, long long ell_cols, int base, V* dense, long long ld,
                                                                int row_major) {
    __shared__ int map[DC_MAPW];
    const long long nbr = (m + bs - 1) / bs, nbc = (n + bs - 1) / bs;
    const V z = zero_value<V>();
    for (long long br = blockIdx.x; br < nbr; br += gridDim.x) {
        const int rows_here = m - br * bs < bs ? (int)(m - br * bs) : bs;
        for (long long bc0 = 0; bc0 < nbc; bc0 += DC_MAPW) {
            const int nb = nbc - bc0 < DC_MAPW ? (int)(nbc - bc0) : DC_MAPW;
            for (int t = threadIdx.x; t < nb; t += DC_THREADS) map[t] = -1;
            __syncthreads();
            for (int k = threadIdx.x; k < eb; k += DC_THREADS) {
                const long long c = (long long)__ldg(colind + br * eb + k) - base;
                if (c >= bc0 && c < bc0 + nb) atomicMax(&map[c - bc0], k);
            }
            __syncthreads();
            const long long j0 = bc0 * bs;
            const long long cols_here = n - j0 < (long long)nb * bs ? n - j0 : (long long)nb * bs;
            const long long total = cols_here * rows_here;
            for (long long t = threadIdx.x; t < total; t += DC_THREADS) {
                const long long r = row_major ? t / cols_here : t % rows_here, c = row_major ? t % cols_here : t / rows_here;
                const long long i = br * bs + r, j = j0 + c;
                const int k = map[c / bs];
                dense[row_major ? i * ld + j : i + j * ld] = k >= 0 ? val[i * ell_cols + (long long)k * bs + j % bs] : z;
            }
            __syncthreads();
        }
    }
}

// one lane's elements of a line found non-zero: write them at the warp's running position, inside [lo, hi) only
template <typename V>
__device__ __forceinline__ void emit(long long pos, long long hi, int j, const V& v, int base, int* ind, V* val) {
    if (pos < hi) {
        ind[pos] = j + base;
        val[pos] = v;
    }
}

// exclusive warp prefix of c, and the warp's total
__device__ __forceinline__ int warp_excl(int c, int lane, int* total) {
    int x = c;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        const int y = __shfl_up_sync(0xffffffffu, x, d);
        if (lane >= d) x += y;
    }
    *total = __shfl_sync(0xffffffffu, x, 31);
    return x - c;
}

template <typename V>
__global__ void __launch_bounds__(DC_THREADS) dense2csr_along_kernel(long long M, long long N, long long nnz, const V* dense, long long ld, int pw,
                                                                     const int* off, int* ind, V* val, int base) {
    constexpr int K = 16 / (int)sizeof(V);
    const int lane = threadIdx.x & 31;
    const long long warps = (long long)gridDim.x * (DC_THREADS / 32);
    for (long long i = (long long)blockIdx.x * (DC_THREADS / 32) + (threadIdx.x >> 5); i < M; i += warps) {
        const V* row = dense + i * ld;
        const long long lo = entry(off, i, base, nnz), hi = entry(off, i + 1, base, nnz);
        long long cnt = 0, j0 = 0;
        if (((uintptr_t)row & 15) == 0) {              // 16-byte vectors of K elements
            const long long nv = N / K;
            for (long long v0 = 0; v0 < nv; v0 += 32) {
                const long long vi = v0 + lane;
                const uint4 x = vi < nv ? __ldg((const uint4*)row + vi) : make_uint4(0, 0, 0, 0);
                unsigned mask = 0;
#pragma unroll
                for (int k = 0; k < K; ++k) mask |= (vi < nv && nonzero(element<V>(x, k), pw)) ? 1u << k : 0u;
                int total;
                long long pos = lo + cnt + warp_excl(__popc(mask), lane, &total);
#pragma unroll
                for (int k = 0; k < K; ++k)
                    if (mask >> k & 1u) emit(pos++, hi, (int)(vi * K + k), element<V>(x, k), base, ind, val);
                cnt += total;
            }
            j0 = nv * K;
        }
        for (; j0 < N; j0 += 32) {                     // scalar: an unaligned line, and the tail of an aligned one
            const long long j = j0 + lane;
            V v;
            const bool p = j < N && nonzero(v = row[j], pw);
            const unsigned b = __ballot_sync(0xffffffffu, p);
            if (p) emit(lo + cnt + __popc(b & ((1u << lane) - 1u)), hi, (int)j, v, base, ind, val);
            cnt += __popc(b);
        }
    }
}

// a CTA of 32 warps per panel of 32 major lines: 32 x 32 tiles staged through shared memory, so the dense reads run along the
// contiguous (major) dimension and each warp then walks its own line across the tile
template <typename V>
__global__ void __launch_bounds__(1024) dense2csr_across_kernel(long long M, long long N, long long nnz, const V* dense, long long ld, int pw,
                                                                const int* off, int* ind, V* val, int base) {
    __shared__ V tile[32][33];
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    for (long long i0 = (long long)blockIdx.x * 32; i0 < M; i0 += (long long)gridDim.x * 32) {
        const bool mine = i0 + w < M;
        const long long lo = mine ? entry(off, i0 + w, base, nnz) : 0, hi = mine ? entry(off, i0 + w + 1, base, nnz) : 0;
        long long cnt = 0;
        for (long long j0 = 0; j0 < N; j0 += 32) {
            if (i0 + lane < M && j0 + w < N) tile[w][lane] = dense[i0 + lane + (j0 + w) * ld];
            __syncthreads();
            const bool act = mine && j0 + lane < N;
            V v;
            if (act) v = tile[lane][w];
            const bool p = act && nonzero(v, pw);
            const unsigned b = __ballot_sync(0xffffffffu, p);
            if (p) emit(lo + cnt + __popc(b & ((1u << lane) - 1u)), hi, (int)(j0 + lane), v, base, ind, val);
            cnt += __popc(b);
            __syncthreads();
        }
    }
}

// dense -> Blocked-ELL, one CTA per block row: every element of the block row's ellValue rows (bs x ell_cols, row-major) from the
// dense block its slot names; a slot whose column lies outside the matrix (the -1 padding among them) is written as zero when
// pad_zero, else left as it is
template <typename V>
__global__ void __launch_bounds__(DC_THREADS) dense2bell_kernel(long long m, long long n, int bs, int eb, const V* dense, long long ld,
                                                                int row_major, const int* colind, V* val, long long ell_cols, int base,
                                                                int pad_zero) {
    const long long nbr = (m + bs - 1) / bs, nbc = (n + bs - 1) / bs;
    const V z = zero_value<V>();
    for (long long br = blockIdx.x; br < nbr; br += gridDim.x) {
        const int rows_here = m - br * bs < bs ? (int)(m - br * bs) : bs;
        const long long total = (long long)rows_here * ell_cols;
        for (long long t = threadIdx.x; t < total; t += DC_THREADS) {
            const long long i = br * bs + t / ell_cols, cc = t % ell_cols;
            const long long bc = (long long)__ldg(colind + br * eb + cc / bs) - base;
            const long long j = bc * bs + cc % bs;
            V* out = val + i * ell_cols + cc;
            if (bc < 0 || bc >= nbc) {
                if (pad_zero) *out = z;
            } else {
                *out = j < n ? dense[row_major ? i * ld + j : i + j * ld] : z;
            }
        }
    }
}

static bool aligned(const void* p, size_t a) { return ((uintptr_t)p & (a - 1)) == 0; }
static bool width_ok(int w) { return w == 2 || w == 4 || w == 8 || w == 16; }
static bool dims_ok(int64_t m, int64_t n) { return m >= 0 && n >= 0 && m <= INT32_MAX - 64 && n <= INT32_MAX - 64; }
static bool order_ok(int order) { return order == ORDER_COL || order == ORDER_ROW; }
// ld of a rows x cols window in this order: at least the contiguous dimension, and at least 1
static bool ld_ok(int64_t rows, int64_t cols, int64_t ld, int order) { return ld >= 1 && ld >= (order == ORDER_ROW ? cols : rows); }

static unsigned grid_for(long long work, long long per_cta) {
    long long g = (work + per_cta - 1) / per_cta;
    if (g > 132 * 32) g = 132 * 32;
    return (unsigned)(g < 1 ? 1 : g);
}

// part width of a dense -> sparse value type (cudaDataType): the width, or half of it for a complex type; 0 for a type the
// predicate does not serve: integers, unknown types, and complex fp16 / bf16, whose predicate was not pinned
static int part_width(int vtype, int* width) {
    switch (vtype) {
    case 2: case 14: *width = 2; return 2;          // CUDA_R_16F, CUDA_R_16BF
    case 0: *width = 4; return 4;                   // CUDA_R_32F
    case 1: *width = 8; return 8;                   // CUDA_R_64F
    case 4: *width = 8; return 4;                   // CUDA_C_32F
    case 5: *width = 16; return 8;                  // CUDA_C_64F
    default: *width = 0; return 0;
    }
}

template <typename V>
static void launch_csr2dense(cudaStream_t st, bool along, long long M, long long N, long long nnz, const int* off, const int* ind, const void* val,
                             int base, void* dense, long long ld) {
    if (along)
        csr2dense_along_kernel<V><<<grid_for(M, DC_THREADS / 32), DC_THREADS, 0, st>>>(M, N, nnz, off, ind, (const V*)val, base, (V*)dense, ld);
    else
        csr2dense_across_kernel<V><<<grid_for(M, DC_PANEL), DC_THREADS, 0, st>>>(M, N, nnz, off, ind, (const V*)val, base, (V*)dense, ld);
}

template <typename V>
static void launch_coo2dense(cudaStream_t st, long long m, long long n, long long nnz, const int* rows, const int* cols, const void* val,
                             int base, void* dense, long long ld, int order) {
    const bool rm = order == ORDER_ROW;
    const long long lines = rm ? m : n, len = rm ? n : m;
    if (lines > 0 && len > 0)
        zero_window_kernel<V><<<grid_for(lines, DC_THREADS / 32), DC_THREADS, 0, st>>>(lines, len, (V*)dense, ld);
    if (nnz > 0)
        coo_scatter_kernel<V><<<grid_for(nnz, DC_THREADS), DC_THREADS, 0, st>>>(m, n, nnz, rows, cols, (const V*)val, base, (V*)dense, ld,
                                                                               (int)rm);
}

template <typename V>
static void launch_bell2dense(cudaStream_t st, long long m, long long n, int bs, int eb, const int* colind, const void* val,
                              long long ell_cols, int base, void* dense, long long ld, int order) {
    bell2dense_kernel<V><<<grid_for((m + bs - 1) / bs, 1), DC_THREADS, 0, st>>>(m, n, bs, eb, colind, (const V*)val, ell_cols, base,
                                                                              (V*)dense, ld, (int)(order == ORDER_ROW));
}

template <typename V>
static void launch_dense2csr(cudaStream_t st, bool along, long long M, long long N, long long nnz, const void* dense, long long ld, int pw,
                             const int* off,
                             int* ind, void* val, int base) {
    if (along)
        dense2csr_along_kernel<V><<<grid_for(M, DC_THREADS / 32), DC_THREADS, 0, st>>>(M, N, nnz, (const V*)dense, ld, pw, off, ind, (V*)val, base);
    else
        dense2csr_across_kernel<V><<<grid_for(M, 32), 1024, 0, st>>>(M, N, nnz, (const V*)dense, ld, pw, off, ind, (V*)val, base);
}

template <typename V>
static void launch_dense2bell(cudaStream_t st, long long m, long long n, int bs, int eb, const void* dense, long long ld, int order,
                              const int* colind, void* val, long long ell_cols, int base) {
    dense2bell_kernel<V><<<grid_for((m + bs - 1) / bs, 1), DC_THREADS, 0, st>>>(m, n, bs, eb, (const V*)dense, ld, (int)(order == ORDER_ROW),
                                                                              colind, (V*)val, ell_cols, base, DC_BELL_PAD_ZERO);
}

#define DC_BY_WIDTH(w, f, ...)                                   \
    switch (w) {                                                 \
    case 2: f<Bits<2>::T>(__VA_ARGS__); break;                   \
    case 4: f<Bits<4>::T>(__VA_ARGS__); break;                   \
    case 8: f<Bits<8>::T>(__VA_ARGS__); break;                   \
    default: f<Bits<16>::T>(__VA_ARGS__); break;                 \
    }

// Blocked-ELL shape: bs >= 1, ell_cols a multiple of bs within the block columns, sizes that fit the kernels' ints
static bool bell_ok(int64_t m, int64_t n, int64_t bs, int64_t ell_cols) {
    if (!dims_ok(m, n) || bs < 1 || bs > 65536 || ell_cols < 0 || ell_cols % bs) return false;
    return ell_cols / bs <= (n + bs - 1) / bs && (m + bs - 1) / bs * (ell_cols / bs) <= INT32_MAX;
}

}  // namespace b200

using namespace b200;

extern "C" {

int b200csr2dense(void* stream, int csc, int64_t m, int64_t n, int64_t nnz, const void* off, const void* ind, const void* val, int value_bytes,
                  int32_t base, void* dense, int64_t ld, int order) {
    if (!dims_ok(m, n) || nnz < 0 || !width_ok(value_bytes) || (base != 0 && base != 1) || !order_ok(order) || !ld_ok(m, n, ld, order))
        return -1;
    if (m == 0 || n == 0) return 0;
    const long long M = csc ? n : m, N = csc ? m : n;
    if (!off || !dense || !aligned(off, 4) || !aligned(dense, value_bytes)) return -1;
    if (nnz > 0 && (!ind || !val || !aligned(ind, 4) || !aligned(val, value_bytes))) return -1;
    const bool along = (order == ORDER_ROW) == !csc;
    DC_BY_WIDTH(value_bytes, launch_csr2dense, (cudaStream_t)stream, along, M, N, (long long)nnz, (const int*)off, (const int*)ind, val, base, dense, ld);
    return (int)cudaGetLastError();
}

int b200coo2dense(void* stream, int64_t m, int64_t n, int64_t nnz, const void* rows, const void* cols, const void* val, int value_bytes,
                  int32_t base, void* dense, int64_t ld, int order) {
    if (!dims_ok(m, n) || nnz < 0 || !width_ok(value_bytes) || (base != 0 && base != 1) || !order_ok(order) || !ld_ok(m, n, ld, order))
        return -1;
    if (m == 0 || n == 0) return 0;
    if (!dense || !aligned(dense, value_bytes)) return -1;
    if (nnz > 0 && (!rows || !cols || !val || !aligned(rows, 4) || !aligned(cols, 4) || !aligned(val, value_bytes))) return -1;
    DC_BY_WIDTH(value_bytes, launch_coo2dense, (cudaStream_t)stream, m, n, nnz, (const int*)rows, (const int*)cols, val, base, dense, ld,
                order);
    return (int)cudaGetLastError();
}

int b200bell2dense(void* stream, int64_t m, int64_t n, int64_t bs, int64_t ell_cols, const void* colind, const void* val, int value_bytes,
                   int32_t base, void* dense, int64_t ld, int order) {
    if (!bell_ok(m, n, bs, ell_cols) || !width_ok(value_bytes) || (base != 0 && base != 1) || !order_ok(order) || !ld_ok(m, n, ld, order))
        return -1;
    if (m == 0 || n == 0) return 0;
    if (!dense || !aligned(dense, value_bytes)) return -1;
    if (ell_cols > 0 && (!colind || !val || !aligned(colind, 4) || !aligned(val, value_bytes))) return -1;
    DC_BY_WIDTH(value_bytes, launch_bell2dense, (cudaStream_t)stream, m, n, (int)bs, (int)(ell_cols / bs), (const int*)colind, val,
                ell_cols, base, dense, ld, order);
    return (int)cudaGetLastError();
}

int b200dense2csr(void* stream, int csc, int64_t m, int64_t n, int64_t nnz, const void* dense, int64_t ld, int order, int value_type,
                  const void* off, void* ind, void* val, int32_t base) {
    int w = 0;
    const int pw = part_width(value_type, &w);
    if (!dims_ok(m, n) || nnz < 0 || pw == 0 || (base != 0 && base != 1) || !order_ok(order) || !ld_ok(m, n, ld, order)) return -1;
    if (m == 0 || n == 0 || nnz == 0) return 0;
    const long long M = csc ? n : m, N = csc ? m : n;
    if (!dense || !off || !ind || !val || !aligned(dense, w) || !aligned(off, 4) || !aligned(ind, 4) || !aligned(val, w)) return -1;
    const bool along = (order == ORDER_ROW) == !csc;
    DC_BY_WIDTH(w, launch_dense2csr, (cudaStream_t)stream, along, M, N, (long long)nnz, dense, ld, pw, (const int*)off, (int*)ind, val, base);
    return (int)cudaGetLastError();
}

int b200dense2bell(void* stream, int64_t m, int64_t n, int64_t bs, int64_t ell_cols, const void* dense, int64_t ld, int order,
                   int value_bytes, const void* colind, void* val, int32_t base) {
    if (!bell_ok(m, n, bs, ell_cols) || !width_ok(value_bytes) || (base != 0 && base != 1) || !order_ok(order) || !ld_ok(m, n, ld, order))
        return -1;
    if (m == 0 || n == 0 || ell_cols == 0) return 0;
    if (!dense || !colind || !val || !aligned(dense, value_bytes) || !aligned(colind, 4) || !aligned(val, value_bytes)) return -1;
    DC_BY_WIDTH(value_bytes, launch_dense2bell, (cudaStream_t)stream, m, n, (int)bs, (int)(ell_cols / bs), dense, ld, order,
                (const int*)colind, val, ell_cols, base);
    return (int)cudaGetLastError();
}

}  // extern "C"
