// spgemm_csr.cu -- the numeric phase of sparse x sparse with structure reuse (cusparseSpGEMMreuse_compute) for CSR on sm_90a:
// C = alpha A B + beta C on a C pattern the closed library's symbolic phase built (include/b200spmv.h, b200spgemm_*).  DESIGN.md 3.28.
//
// The plan (b200spgemm_plan, once per pattern) checks the three patterns on the device, counts the products of every C row
// (sum over A row i's k of nnz(B row k)) and cuts every C row into windows of at most kWindow stored columns.  Each window is one
// "pass" for one warp; the passes are listed heaviest bin first, so the compute kernel's dynamic queue starts the hub rows early.
//
// Compute: a warp takes a pass, stages the window's C columns in shared memory and zeroes one accumulator per column.  It walks
// A row i in stored order; for each (i, k) the lanes stride B row k, find each column j in the window by binary search and add
// a_ik * b_kj into j's slot.  The columns of one B row are distinct, so no two lanes share a slot in a step, and __syncwarp()
// orders the steps of successive k.  Every C(i, j) is therefore the left fold over A's stored order of correctly rounded
// products, acc = fadd(acc, fmul(a_ik, b_kj)) from acc = +0, whatever the window, bin or launch: long rows (several windows, each
// re-walking A row i) give the same bits as short ones.  No atomics on values, no allocation, no host synchronisation.
#include <cuda_runtime.h>

#include <algorithm>
#include <climits>
#include <cstdint>

#include "../../include/b200spmv.h"
#include "spmv_common.cuh"

namespace b200 {

constexpr int kSpgemmWindow = 256;        // C columns one warp stages: 256 * (4 + 8) B = 3 KB per warp in fp64
constexpr int kSpgemmWarps = 8;           // warps per CTA of both kernels
constexpr int kSpgemmBins = 4;
constexpr int kSpgemmCtasPerSm = 8;       // the compute grid: 8 x 8 warps per SM (64, the most an SM holds)
// products-per-row edges of the bins, heaviest first: bin 0 >= 2^14, bin 1 >= 2^10, bin 2 >= 2^6, bin 3 the rest
__host__ __device__ constexpr long long spgemm_bin_edge(int b) { return b == 0 ? (1LL << 14) : (b == 1 ? (1LL << 10) : (1LL << 6)); }

// plan header: 64-bit words
enum { SG_BAD = 0, SG_MISSING = 1, SG_QUEUE = 2, SG_PASSES = 3, SG_BIN_COUNT = 4, SG_BIN_FILL = 8, SG_WORDS = 12 };

struct SpgemmLayout {
    size_t npass, bin, passes, total;
};
static SpgemmLayout spgemm_layout(int64_t rows, int64_t nnz_c) {
    SpgemmLayout l;
    const size_t max_passes = (size_t)rows + (size_t)nnz_c / kSpgemmWindow + 1;
    l.npass = 256;
    l.bin = l.npass + round_up_256(4 * (size_t)rows);
    l.passes = l.bin + round_up_256(4 * (size_t)rows);
    l.total = l.passes + round_up_256(8 * max_passes);
    return l;
}

__device__ __forceinline__ int spgemm_bin_of(long long work) {
    return work >= spgemm_bin_edge(0) ? 0 : (work >= spgemm_bin_edge(1) ? 1 : (work >= spgemm_bin_edge(2) ? 2 : 3));
}

// One warp per row: check C row i (offsets inside [0, nnz_c], non-decreasing, columns strictly ascending inside [0, cols)), A row
// i (offsets as C's, columns inside [0, krows)) and the B rows it names (offsets inside [0, nnz_b], non-decreasing), then count
// the row's products.  A bad row sets its bit in hdr[SG_BAD] and reads nothing past what it checked.
__global__ void __launch_bounds__(kSpgemmWarps * 32)
spgemm_plan_rows_kernel(int rows, int krows, int cols, long long nnz_a, long long nnz_b, long long nnz_c, const int* __restrict__ a_off,
                        const int* __restrict__ a_col, int a_base, const int* __restrict__ b_off, int b_base,
                        const int* __restrict__ c_off, const int* __restrict__ c_col, int c_base, unsigned long long* hdr,
                        int* __restrict__ npass, int* __restrict__ bin) {
    const int lane = threadIdx.x & 31;
    for (long long i = (long long)blockIdx.x * kSpgemmWarps + (threadIdx.x >> 5); i < rows; i += (long long)gridDim.x * kSpgemmWarps) {
        unsigned flags = 0;
        const long long c0 = (long long)c_off[i] - c_base, c1 = (long long)c_off[i + 1] - c_base;
        if (c0 < 0 || c0 > c1 || c1 > nnz_c || (i == 0 && c0 != 0) || (i == rows - 1 && c1 != nnz_c)) flags |= 1u;
        const long long a0 = (long long)a_off[i] - a_base, a1 = (long long)a_off[i + 1] - a_base;
        if (a0 < 0 || a0 > a1 || a1 > nnz_a) flags |= 4u;
        if (!(flags & 1u))
            for (long long p = c0 + lane; p < c1; p += 32) {
                const long long j = (long long)c_col[p] - c_base;
                if (j < 0 || j >= cols || (p > c0 && (long long)c_col[p - 1] - c_base >= j)) flags |= 2u;
            }
        long long work = 0;
        if (!(flags & 4u))
            for (long long p = a0 + lane; p < a1; p += 32) {
                const long long k = (long long)a_col[p] - a_base;
                if (k < 0 || k >= krows) { flags |= 4u; continue; }
                const long long b0 = (long long)b_off[k] - b_base, b1 = (long long)b_off[k + 1] - b_base;
                if (b0 < 0 || b0 > b1 || b1 > nnz_b) flags |= 8u;
                else work += b1 - b0;
            }
        flags = __reduce_or_sync(0xffffffffu, flags);
        work = warp_allsum(work);
        if (lane == 0) {
            int n = 0, b = 0;
            if (flags) atomicOr(hdr + SG_BAD, (unsigned long long)flags);
            else if (c1 > c0) {
                n = (int)((c1 - c0 + kSpgemmWindow - 1) / kSpgemmWindow);
                b = spgemm_bin_of(work);
                atomicAdd(hdr + SG_BIN_COUNT + b, (unsigned long long)n);
            }
            npass[i] = n;
            bin[i] = b;
        }
    }
}

// Lists every row's passes {row, window} in its bin's range, bins heaviest first (the order inside a bin is the order of arrival:
// no result depends on it).  Runs only on a plan whose patterns all passed.
__global__ void __launch_bounds__(256)
spgemm_plan_passes_kernel(int rows, unsigned long long* hdr, const int* __restrict__ npass, const int* __restrict__ bin,
                          int2* __restrict__ passes) {
    if (hdr[SG_BAD]) return;
    unsigned long long start[kSpgemmBins], total = 0;
#pragma unroll
    for (int b = 0; b < kSpgemmBins; ++b) { start[b] = total; total += hdr[SG_BIN_COUNT + b]; }
    if (blockIdx.x == 0 && threadIdx.x == 0) hdr[SG_PASSES] = total;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < rows; i += (long long)gridDim.x * blockDim.x) {
        const int n = npass[i];
        if (n == 0) continue;
        const int b = bin[i];
        const unsigned long long pos = start[b] + atomicAdd(hdr + SG_BIN_FILL + b, (unsigned long long)n);
        for (int q = 0; q < n; ++q) passes[pos + q] = make_int2((int)i, q);
    }
}

// first position of a window column >= j (width when none)
__device__ __forceinline__ int spgemm_lower_bound(const int* s, int width, int j) {
    int lo = 0, hi = width;
    while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (s[mid] < j) lo = mid + 1; else hi = mid;
    }
    return lo;
}

__device__ __forceinline__ float mul_rn(float a, float b) { return __fmul_rn(a, b); }
__device__ __forceinline__ double mul_rn(double a, double b) { return __dmul_rn(a, b); }
__device__ __forceinline__ float add_rn(float a, float b) { return __fadd_rn(a, b); }
__device__ __forceinline__ double add_rn(double a, double b) { return __dadd_rn(a, b); }

template <typename T>
__global__ void __launch_bounds__(kSpgemmWarps * 32)
spgemm_compute_kernel(const int* __restrict__ a_off, const int* __restrict__ a_col, const T* __restrict__ a_val, int a_base,
                      const int* __restrict__ b_off, const int* __restrict__ b_col, const T* __restrict__ b_val, int b_base,
                      const int* __restrict__ c_off, const int* __restrict__ c_col, T* __restrict__ c_val, int c_base, Scalars<T> s,
                      unsigned long long* hdr, const int* __restrict__ npass, const int2* __restrict__ passes) {
    __shared__ int s_col[kSpgemmWarps][kSpgemmWindow];
    __shared__ T s_acc[kSpgemmWarps][kSpgemmWindow];
    const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
    int* col = s_col[w];
    T* acc = s_acc[w];
    const unsigned long long total = hdr[SG_PASSES];
    const T alpha = s.a(), beta = s.b();
    for (;;) {
        unsigned long long g = 0;
        if (lane == 0) g = atomicAdd(hdr + SG_QUEUE, 1ULL);
        g = __shfl_sync(0xffffffffu, g, 0);
        if (g >= total) break;
        const int2 pr = passes[g];
        const int i = pr.x, q = pr.y, n = npass[i];
        const long long c0 = (long long)c_off[i] - c_base, len = (long long)c_off[i + 1] - c_base - c0;
        const long long p0 = len * q / n, p1 = len * (q + 1) / n;
        const int width = (int)(p1 - p0);
        for (int t = lane; t < width; t += 32) {
            col[t] = c_col[c0 + p0 + t] - c_base;
            acc[t] = T(0);
        }
        __syncwarp();
        // the columns this window answers for: from its first (or -inf) to the next window's first (or +inf); a j between two
        // windows is claimed by the earlier one, so each missing product is counted once
        const int lo = q == 0 ? INT_MIN : col[0];
        const int hi = q == n - 1 ? INT_MAX : c_col[c0 + p1] - c_base;
        unsigned missing = 0;
        const long long a0 = (long long)a_off[i] - a_base, a1 = (long long)a_off[i + 1] - a_base;
        for (long long ab = a0; ab < a1; ab += 32) {
            // 32 entries of A row i at once: each lane holds one (k, a_ik) and B row k's range, broadcast in stored order below
            int my_b0 = 0, my_b1 = 0;
            T my_a = T(0);
            if (ab + lane < a1) {
                const int k = a_col[ab + lane] - a_base;
                my_a = a_val[ab + lane];
                my_b0 = b_off[k] - b_base;
                my_b1 = b_off[k + 1] - b_base;
            }
            const int m = (int)min(32LL, a1 - ab);
            for (int t = 0; t < m; ++t) {
                const T av = __shfl_sync(0xffffffffu, my_a, t);
                const int b0 = __shfl_sync(0xffffffffu, my_b0, t), b1 = __shfl_sync(0xffffffffu, my_b1, t);
                for (int e = b0 + lane; e < b1; e += 32) {
                    const int j = b_col[e] - b_base;
                    if (j < lo || j >= hi) continue;
                    const int pos = spgemm_lower_bound(col, width, j);
                    if (pos < width && col[pos] == j) acc[pos] = add_rn(acc[pos], mul_rn(av, b_val[e]));
                    else ++missing;
                }
                __syncwarp();
            }
        }
        for (int t = lane; t < width; t += 32) {
            const long long p = c0 + p0 + t;
            T v = mul_rn(alpha, acc[t]);
            if (beta != T(0)) v = add_rn(v, mul_rn(beta, c_val[p]));      // beta = 0 never reads C (it may hold NaN)
            c_val[p] = v;
        }
        missing = __reduce_add_sync(0xffffffffu, missing);
        if (lane == 0 && missing) atomicAdd(hdr + SG_MISSING, (unsigned long long)missing);
        __syncwarp();                                                     // the window is restaged by the next pass
    }
}

template <typename T>
static int spgemm_launch(cudaStream_t stream, int64_t rows, int64_t nnz_c, const void* a_off, const void* a_col, const void* a_val,
                         int a_base, const void* b_off, const void* b_col, const void* b_val, int b_base, const void* c_off,
                         const void* c_col, void* c_val, int c_base, const void* alpha, const void* beta, int on_dev, void* plan) {
    const SpgemmLayout l = spgemm_layout(rows, nnz_c);
    char* p = (char*)plan;
    unsigned long long* hdr = (unsigned long long*)p;
    Scalars<T> s;
    set_scalars(s, alpha, beta, on_dev);
    cudaError_t e = cudaMemsetAsync(hdr + SG_QUEUE, 0, sizeof(unsigned long long), stream);
    if (e != cudaSuccess) return (int)e;
    int dev = 0, sms = 0;
    if ((e = cudaGetDevice(&dev)) != cudaSuccess || (e = cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev)) != cudaSuccess)
        return (int)e;
    const long long bound = rows + nnz_c / kSpgemmWindow + 1;        // the most passes a plan of these sizes lists
    const long long ctas = std::min<long long>((bound + kSpgemmWarps - 1) / kSpgemmWarps, (long long)sms * kSpgemmCtasPerSm);
    spgemm_compute_kernel<T><<<(unsigned)std::max(ctas, 1LL), kSpgemmWarps * 32, 0, stream>>>(
        (const int*)a_off, (const int*)a_col, (const T*)a_val, a_base, (const int*)b_off, (const int*)b_col, (const T*)b_val, b_base,
        (const int*)c_off, (const int*)c_col, (T*)c_val, c_base, s, hdr, (const int*)(p + l.npass), (const int2*)(p + l.passes));
    return (int)cudaGetLastError();
}

}  // namespace b200

using namespace b200;

static bool spgemm_sizes_ok(int64_t rows, int64_t krows, int64_t cols, int64_t nnz_a, int64_t nnz_b, int64_t nnz_c) {
    return rows >= 0 && rows < INT32_MAX && krows >= 0 && krows < INT32_MAX && cols >= 0 && cols < INT32_MAX && nnz_a >= 0 &&
           nnz_a < INT32_MAX && nnz_b >= 0 && nnz_b < INT32_MAX && nnz_c >= 0 && nnz_c < INT32_MAX;
}

extern "C" {

size_t b200spgemm_plan_size(int64_t rows, int64_t nnz_a, int64_t nnz_b, int64_t nnz_c) {
    (void)nnz_a; (void)nnz_b;
    if (rows < 0 || nnz_c < 0) return 0;
    return spgemm_layout(rows, nnz_c).total;
}

void b200spgemm_params(int32_t* window, int32_t* warps_per_cta, int64_t* bin_edges) {
    if (window) *window = kSpgemmWindow;
    if (warps_per_cta) *warps_per_cta = kSpgemmWarps;
    if (bin_edges)
        for (int b = 0; b < kSpgemmBins - 1; ++b) bin_edges[b] = spgemm_bin_edge(b);
}

int b200spgemm_plan(void* stream, int64_t rows, int64_t krows, int64_t cols, int64_t nnz_a, int64_t nnz_b, int64_t nnz_c,
                    const void* a_off, const void* a_col, int32_t a_base, const void* b_off, int32_t b_base, const void* c_off,
                    const void* c_col, int32_t c_base, void* plan, size_t plan_bytes, int64_t* passes, uint64_t* bad) {
    if (!spgemm_sizes_ok(rows, krows, cols, nnz_a, nnz_b, nnz_c) || (a_base | b_base | c_base) & ~1) return -1;
    if (!workspace_usable(plan, plan_bytes, b200spgemm_plan_size(rows, nnz_a, nnz_b, nnz_c))) return -1;
    if (rows > 0 && (!a_off || !b_off || !c_off || (nnz_a > 0 && !a_col) || (nnz_c > 0 && !c_col))) return -1;
    cudaStream_t st = (cudaStream_t)stream;
    const SpgemmLayout l = spgemm_layout(rows, nnz_c);
    char* p = (char*)plan;
    unsigned long long* hdr = (unsigned long long*)p;
    cudaError_t e = cudaMemsetAsync(hdr, 0, SG_WORDS * sizeof(unsigned long long), st);
    if (e != cudaSuccess) return (int)e;
    if (rows > 0) {
        const long long ctas = std::min<long long>((rows + kSpgemmWarps - 1) / kSpgemmWarps, 1LL << 16);
        spgemm_plan_rows_kernel<<<(unsigned)ctas, kSpgemmWarps * 32, 0, st>>>(
            (int)rows, (int)krows, (int)cols, nnz_a, nnz_b, nnz_c, (const int*)a_off, (const int*)a_col, a_base, (const int*)b_off,
            b_base, (const int*)c_off, (const int*)c_col, c_base, hdr, (int*)(p + l.npass), (int*)(p + l.bin));
        if ((e = cudaGetLastError()) != cudaSuccess) return (int)e;
        spgemm_plan_passes_kernel<<<(unsigned)std::min<long long>((rows + 255) / 256, 1LL << 16), 256, 0, st>>>(
            (int)rows, hdr, (const int*)(p + l.npass), (const int*)(p + l.bin), (int2*)(p + l.passes));
        if ((e = cudaGetLastError()) != cudaSuccess) return (int)e;
    }
    unsigned long long h[SG_WORDS] = {};
    if ((e = cudaMemcpyAsync(h, hdr, sizeof(h), cudaMemcpyDeviceToHost, st)) != cudaSuccess) return (int)e;
    if ((e = cudaStreamSynchronize(st)) != cudaSuccess) return (int)e;
    if (bad) *bad = h[SG_BAD];
    if (passes) *passes = (int64_t)h[SG_PASSES];
    return h[SG_BAD] ? B200SPGEMM_BAD_PATTERN : 0;
}

int b200spgemm_compute(void* stream, int dtype, int64_t rows, int64_t nnz_c, const void* a_off, const void* a_col, const void* a_val,
                       int32_t a_base, const void* b_off, const void* b_col, const void* b_val, int32_t b_base, const void* c_off,
                       const void* c_col, void* c_val, int32_t c_base, const void* alpha, const void* beta, int scalars_on_device,
                       void* plan) {
    if ((dtype != 0 && dtype != 1) || rows < 0 || rows >= INT32_MAX || nnz_c < 0 || nnz_c >= INT32_MAX || !plan || !alpha || !beta ||
        (a_base | b_base | c_base) & ~1)
        return -1;
    if (rows == 0) return 0;
    return dtype == 1 ? spgemm_launch<double>((cudaStream_t)stream, rows, nnz_c, a_off, a_col, a_val, a_base, b_off, b_col, b_val, b_base,
                                              c_off, c_col, c_val, c_base, alpha, beta, scalars_on_device, plan)
                      : spgemm_launch<float>((cudaStream_t)stream, rows, nnz_c, a_off, a_col, a_val, a_base, b_off, b_col, b_val, b_base,
                                             c_off, c_col, c_val, c_base, alpha, beta, scalars_on_device, plan);
}

}  // extern "C"
