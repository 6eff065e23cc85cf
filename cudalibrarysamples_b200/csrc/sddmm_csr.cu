// sddmm_csr.cu -- sampled dense-dense product  C = alpha * (op(A) * op(B)) o spy(C) + beta * C  on H100 (sm_90a), C in CSR
// (int32 offsets / columns), A and B dense, fp32 / fp64.  Replaces the closed library behind cusparseSDDMM
// (cuSPARSE/sddmm_csr/sddmm_csr_example.c:114-134, cuSPARSE/sddmm_csr_batched/sddmm_csr_batched_example.c:146-166).
//
// Every layout is reduced to element strides: op(A)(i, k) = A[i * sai + k * sak], op(B)(k, j) = B[k * sbk + j * sbj], so one
// kernel serves all 16 combinations of order and op.  Each entry of C is one dot product of length K, independent of all the
// others: no reduction crosses a warp, no atomics, no fix-up launch, every value of C written exactly once.
//
//   * Work split: flat over the non-zeros.  Warp w owns SDDMM_CHUNK consecutive entries; the row of its first entry comes from
//     one binary search over the offsets, after that each lane walks forward as its entry index grows (csr_transpose_kernel
//     does the same).  R-MAT rows of 10^4-10^5 entries are spread over many warps.
//   * Inside a warp, G lanes (a power of two picked from K) share one entry: lane g of the group takes elements g*V, g*V + G*V,
//     ... of the dot product, and a fixed xor-shuffle tree adds the G partial sums, so the bits do not depend on timing.  Lanes
//     at or beyond K neither load nor multiply, and nothing is read for rows of A / columns of B that C does not reference: a
//     NaN there, or in the padding of a leading dimension, cannot reach C.
//   * V: with K contiguous in both operands (sak == sbk == 1), 16-byte alignment and K a multiple of the vector width, each lane
//     loads V = 16 / sizeof(T) elements per instruction; otherwise V = 1 with strided scalar loads.
//   * An operand that is not K-contiguous (the sddmm_csr sample's B: K x N row-major, NON_TRANSPOSE) is first copied, per call,
//     into the caller's buffer as a tight K-contiguous matrix by spmm_transpose_b_kernel (spmm_csr.cu).  A NULL, misaligned or
//     too small buffer leaves it in place and the strided loads serve it.
//   * A strided batch is one launch: the batch index is blockIdx.y.
// No tensor cores: a sampled product of random pattern has no dense tiles to feed them.
#include "spmv_common.cuh"
#include "config.h"
#include "../../include/b200spmv.h"

namespace b200 {

int transpose_col_to_row_major(cudaStream_t stream, int dtype, const void* B, int64_t ldb, void* Bt, int64_t cols, int64_t n);

constexpr int SDDMM_WARPS = 8;           // warps per CTA
constexpr int SDDMM_CHUNK = 128;         // consecutive non-zeros per warp
constexpr int SDDMM_UNROLL = 4;          // entries a lane group has in flight at once
constexpr int SDDMM_VEC_BYTES = 16;      // width of one vector load on the K-contiguous path

template <typename T>
struct SddmmArgs {
    const int* off;
    const int* col;
    T*         val;
    const T*   A;
    const T*   B;
    int        base, rows, nnz, k, lg;       // lg: log2 of the lane-group width G
    long long  sai, sak, sbk, sbj;           // element strides of op(A)(i, k) and op(B)(k, j)
    long long  off_stride, cv_stride, a_stride, b_stride;   // element strides between the matrices of a batch (0 = shared)
    Scalars<T> s;
};

__device__ __forceinline__ void ldv(const float* p, float (&v)[1]) { v[0] = __ldg(p); }
__device__ __forceinline__ void ldv(const double* p, double (&v)[1]) { v[0] = __ldg(p); }
__device__ __forceinline__ void ldv(const float* p, float (&v)[4]) {
    const float4 q = __ldg((const float4*)p);
    v[0] = q.x; v[1] = q.y; v[2] = q.z; v[3] = q.w;
}
__device__ __forceinline__ void ldv(const double* p, double (&v)[2]) {
    const double2 q = __ldg((const double2*)p);
    v[0] = q.x; v[1] = q.y;
}

// V = 1: strided scalar loads; V = 16 / sizeof(T): K-contiguous vector loads (sak == sbk == 1, checked on the host).
template <typename T, int V>
__global__ void __launch_bounds__(32 * SDDMM_WARPS) sddmm_csr_kernel(const SddmmArgs<T> a) {
    const int lane = (int)threadIdx.x & 31;
    const long long c0 = ((long long)blockIdx.x * SDDMM_WARPS + ((int)threadIdx.x >> 5)) * SDDMM_CHUNK;
    if (c0 >= a.nnz) return;                                       // warp-uniform
    const int n0 = (int)c0, n1 = min(n0 + SDDMM_CHUNK, a.nnz);
    const long long bi = blockIdx.y;
    const int* off = a.off + bi * a.off_stride;
    const int* col = a.col + bi * a.cv_stride;
    T*         val = a.val + bi * a.cv_stride;
    const T*   A = a.A + bi * a.a_stride;
    const T*   B = a.B + bi * a.b_stride;
    // row of entry n0: the last r with off[r] - base <= n0 (invariant off[lo] - base <= n0 < off[hi] - base, off[rows] = nnz).
    // Not csr_row_of: as a call, a.base is loaded ahead of the search and the kernel compiles to different SASS.
    int lo = 0, hi = a.rows;
    while (hi - lo > 1) {
        const int mid = (lo + hi) >> 1;
        if (__ldg(off + mid) - a.base <= n0) lo = mid; else hi = mid;
    }
    int r = lo, rend = __ldg(off + r + 1) - a.base;
    const int G = 1 << a.lg, E = 32 >> a.lg;                       // lanes per entry, entries per warp step
    const int slot = lane >> a.lg, g = lane & (G - 1);
    const long long ska = V == 1 ? a.sak : 1, skb = V == 1 ? a.sbk : 1;
    const T alpha = a.s.a(), beta = a.s.b();
    for (int e0 = n0; e0 < n1; e0 += E * SDDMM_UNROLL) {           // warp-uniform trip count: the shuffles below see every lane
        int      e[SDDMM_UNROLL];
        bool     live[SDDMM_UNROLL];
        const T* pa[SDDMM_UNROLL];
        const T* pb[SDDMM_UNROLL];
#pragma unroll
        for (int u = 0; u < SDDMM_UNROLL; u++) {
            e[u] = e0 + u * E + slot;
            live[u] = e[u] < n1;
            pa[u] = A;
            pb[u] = B;
            if (live[u]) {
                while (rend <= e[u] && r + 1 < a.rows) { r++; rend = __ldg(off + r + 1) - a.base; }
                pa[u] = A + (long long)r * a.sai;
                pb[u] = B + (long long)(ldg_stream(col + e[u]) - a.base) * a.sbj;
            }
        }
        T acc[SDDMM_UNROLL];
#pragma unroll
        for (int u = 0; u < SDDMM_UNROLL; u++) acc[u] = T(0);
        for (int k = g * V; k < a.k; k += G * V) {
            T xa[SDDMM_UNROLL][V], xb[SDDMM_UNROLL][V];
#pragma unroll
            for (int u = 0; u < SDDMM_UNROLL; u++)
                if (live[u]) { ldv(pa[u] + k * ska, xa[u]); ldv(pb[u] + k * skb, xb[u]); }
#pragma unroll
            for (int u = 0; u < SDDMM_UNROLL; u++)
                if (live[u]) {
#pragma unroll
                    for (int v = 0; v < V; v++) acc[u] += xa[u][v] * xb[u][v];
                }
        }
#pragma unroll
        for (int u = 0; u < SDDMM_UNROLL; u++)
            for (int o = G >> 1; o > 0; o >>= 1) acc[u] += __shfl_xor_sync(0xffffffffu, acc[u], o);
#pragma unroll
        for (int u = 0; u < SDDMM_UNROLL; u++)
            if (live[u] && g == 0) val[e[u]] = axpby(alpha, acc[u], beta, val + e[u]);
    }
}

// Transposed copies the call makes in the workspace: an operand whose k stride is not 1 but whose other stride is (a dense
// matrix stored the "wrong" way round for this product) becomes a tight K-contiguous copy, one per matrix of the batch it has.
struct SddmmCopies {
    bool   a = false, b = false;
    size_t a_bytes = 0, b_bytes = 0;
};

static SddmmCopies sddmm_copies(int dtype, int64_t m, int64_t n, int64_t k, int64_t sai, int64_t sak, int64_t sbk, int64_t sbj, int batch,
                                int64_t a_stride, int64_t b_stride) {
    SddmmCopies c;
    const size_t vsz = dtype == 1 ? 8 : 4;
    if (k > 1 && sak != 1 && sai == 1 && m > 0) {
        c.a = true;
        c.a_bytes = round_up_256((size_t)(batch > 1 && a_stride != 0 ? batch : 1) * (size_t)m * (size_t)k * vsz);
    }
    if (k > 1 && sbk != 1 && sbj == 1 && n > 0) {
        c.b = true;
        c.b_bytes = round_up_256((size_t)(batch > 1 && b_stride != 0 ? batch : 1) * (size_t)n * (size_t)k * vsz);
    }
    return c;
}

static int group_log2(int64_t k, int v) {
    const int64_t need = (k + v - 1) / v;                        // lanes one pass over K takes
    int lg = 0;
    while (lg < 5 && (1LL << lg) < need) lg++;
    return lg;
}

template <typename T>
static int launch_sddmm(cudaStream_t stream, int64_t m, int64_t n, int64_t k, int64_t nnz, const void* off, const void* col, void* val,
                        int base, const void* alpha, const void* beta, int on_device, const void* A, int64_t sai, int64_t sak,
                        const void* B, int64_t sbk, int64_t sbj, int batch, int64_t off_stride, int64_t cv_stride, int64_t a_stride,
                        int64_t b_stride, void* ws, size_t ws_bytes) {
    if (k <= 1) { sak = 1; sbk = 1; }                            // a single k: its stride is never used
    if (batch == 1) { off_stride = cv_stride = a_stride = b_stride = 0; }
    const SddmmCopies cp = sddmm_copies(sizeof(T) == 8 ? 1 : 0, m, n, k, sai, sak, sbk, sbj, batch, a_stride, b_stride);
    if ((cp.a || cp.b) && workspace_usable(ws, ws_bytes, cp.a_bytes + cp.b_bytes)) {
        const int dt = sizeof(T) == 8 ? 1 : 0;
        if (cp.a) {
            const int cnt = a_stride != 0 ? batch : 1;
            for (int i = 0; i < cnt; i++) {
                const int rc = transpose_col_to_row_major(stream, dt, (const T*)A + (size_t)i * a_stride, sak, (T*)ws + (size_t)i * m * k, m, k);
                if (rc != 0) return rc;
            }
            A = ws; sai = k; sak = 1; a_stride = a_stride != 0 ? m * k : 0;
        }
        if (cp.b) {
            T* wb = (T*)((char*)ws + cp.a_bytes);
            const int cnt = b_stride != 0 ? batch : 1;
            for (int i = 0; i < cnt; i++) {
                const int rc = transpose_col_to_row_major(stream, dt, (const T*)B + (size_t)i * b_stride, sbk, wb + (size_t)i * n * k, n, k);
                if (rc != 0) return rc;
            }
            B = wb; sbj = k; sbk = 1; b_stride = b_stride != 0 ? n * k : 0;
        }
    }
    constexpr int VW = SDDMM_VEC_BYTES / sizeof(T);
    const bool vec = k > 0 && sak == 1 && sbk == 1 && k % VW == 0 && ((uintptr_t)A & 15) == 0 && ((uintptr_t)B & 15) == 0 &&
                     sai % VW == 0 && sbj % VW == 0 && a_stride % VW == 0 && b_stride % VW == 0;
    SddmmArgs<T> a;
    a.off = (const int*)off; a.col = (const int*)col; a.val = (T*)val; a.A = (const T*)A; a.B = (const T*)B;
    a.base = base; a.rows = (int)m; a.nnz = (int)nnz; a.k = (int)k; a.lg = group_log2(k, vec ? VW : 1);
    a.sai = sai; a.sak = sak; a.sbk = sbk; a.sbj = sbj;
    a.off_stride = off_stride; a.cv_stride = cv_stride; a.a_stride = a_stride; a.b_stride = b_stride;
    set_scalars(a.s, alpha, beta, on_device);
    const int64_t per_cta = (int64_t)SDDMM_CHUNK * SDDMM_WARPS;
    const dim3 grid((unsigned)((nnz + per_cta - 1) / per_cta), (unsigned)batch);
    if (vec) sddmm_csr_kernel<T, VW><<<grid, 32 * SDDMM_WARPS, 0, stream>>>(a);
    else sddmm_csr_kernel<T, 1><<<grid, 32 * SDDMM_WARPS, 0, stream>>>(a);
    return (int)cudaGetLastError();
}

}  // namespace b200

using namespace b200;

extern "C" {

void b200sddmm_params(int32_t* warp_chunk, int32_t* entries_per_group, int32_t* vec_bytes, int32_t* max_group) {
    if (warp_chunk) *warp_chunk = SDDMM_CHUNK;
    if (entries_per_group) *entries_per_group = SDDMM_UNROLL;
    if (vec_bytes) *vec_bytes = SDDMM_VEC_BYTES;
    if (max_group) *max_group = 32;
}

size_t b200sddmm_csr_workspace_bytes(int dtype, int64_t m, int64_t n, int64_t k, int64_t sai, int64_t sak, int64_t sbk, int64_t sbj,
                                     int batch, int64_t a_stride, int64_t b_stride) {
    if ((dtype != 0 && dtype != 1) || m < 0 || n < 0 || k < 0 || batch < 1) return 0;
    if (k <= 1) { sak = 1; sbk = 1; }
    const SddmmCopies c = sddmm_copies(dtype, m, n, k, sai, sak, sbk, sbj, batch, batch > 1 ? a_stride : 0, batch > 1 ? b_stride : 0);
    return c.a_bytes + c.b_bytes;
}

int b200sddmm_csr(void* stream, int dtype, int64_t m, int64_t n, int64_t k, int64_t nnz, const void* row_offsets, const void* col_ind,
                  void* values, int32_t base, const void* alpha, const void* beta, int scalars_on_device, const void* A, int64_t sai,
                  int64_t sak, const void* B, int64_t sbk, int64_t sbj, int batch, int64_t off_stride, int64_t colval_stride,
                  int64_t a_stride, int64_t b_stride, void* workspace, size_t workspace_bytes) {
    if (dtype != 0 && dtype != 1) return -1;
    if (m < 0 || n < 0 || k < 0 || nnz < 0 || !alpha || !beta || (base != 0 && base != 1)) return -1;
    if (batch < 1 || batch > 65535) return -1;
    if (sai < 0 || sak < 0 || sbk < 0 || sbj < 0 || off_stride < 0 || colval_stride < 0 || a_stride < 0 || b_stride < 0) return -1;
    if (m > INT32_MAX - 64 || n > INT32_MAX - 64 || k > INT32_MAX - 64 || nnz > INT32_MAX - 65536) return -1;
    if (m == 0 && nnz > 0) return -1;
    if (batch > 1 && colval_stride < nnz) return -1;             // the batch's outputs would overlap
    if (m == 0 || nnz == 0) return 0;
    if (!row_offsets || !col_ind || !values || (k > 0 && (!A || !B))) return -1;
    if (dtype == 0)
        return launch_sddmm<float>((cudaStream_t)stream, m, n, k, nnz, row_offsets, col_ind, values, base, alpha, beta, scalars_on_device, A,
                                   sai, sak, B, sbk, sbj, batch, off_stride, colval_stride, a_stride, b_stride, workspace, workspace_bytes);
    return launch_sddmm<double>((cudaStream_t)stream, m, n, k, nnz, row_offsets, col_ind, values, base, alpha, beta, scalars_on_device, A,
                                sai, sak, B, sbk, sbj, batch, off_stride, colval_stride, a_stride, b_stride, workspace, workspace_bytes);
}

}  // extern "C"
