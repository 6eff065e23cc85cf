// convert.cu -- sparse format conversions on H100 (sm_90a), int32 indices: CSR -> CSC (cusparseCsr2cscEx2), the in-place COO sort
// (cusparseXcoosortByRow / ByColumn), COO row indices <-> CSR row offsets (cusparseXcoo2csr / Xcsr2coo) and the identity
// permutation (cusparseCreateIdentityPermutation).  DESIGN.md 3.23.
//
// All of it runs on the stable LSD radix sort of the transposed plan (radix_sort.cuh, spmm_csr_t.cu), so every result is a pure
// function of the input, ties included:
//   csr2csc   sorts the entry indices by column: within a column rows ascend, and duplicate (row, col) entries keep their CSR order.
//             The sorted columns give the column pointers, a binary search over the row offsets each entry's row, and the values
//             move by the sorted indices, bit for bit, 1 to 16 bytes wide.  Columns need not be sorted within a row.
//   coosort   sorts by the second key, then by the first key read through that permutation: (row, col) or (col, row) order, equal
//             pairs in input order.  rows, cols and P are then permuted in place, P_out[i] = P_in[sigma(i)].  Keys are plain ints
//             in [0, m] / [0, n] (base 0 and base 1 alike).
// Whatever the indices hold, nothing is written outside the caller's outputs and workspace; the result of out-of-range input is
// undefined.  No allocation, no host synchronisation: graph-capturable.
#include "radix_sort.cuh"
#include "spmv_common.cuh"
#include "../../include/b200spmv.h"

#include <algorithm>

namespace b200 {

__global__ void __launch_bounds__(RT_THREADS) identity_permutation_kernel(int* p, int n) {
    for (long long i = (long long)blockIdx.x * RT_THREADS + threadIdx.x; i < n; i += (long long)gridDim.x * RT_THREADS) p[i] = (int)i;
}

static bool aligned(const void* p, size_t a) { return ((uintptr_t)p & (a - 1)) == 0; }
static bool width_ok(int w) { return w == 1 || w == 2 || w == 4 || w == 8 || w == 16; }

// sizes the sort takes: every key range and entry count fits an int, with room for the last tile
static bool conv_dims_ok(int64_t m, int64_t n, int64_t nnz) {
    return m >= 0 && n >= 0 && nnz >= 0 && m <= INT32_MAX - 64 && n <= INT32_MAX - 64 && nnz <= INT32_MAX - 65536;
}

}  // namespace b200

using namespace b200;

extern "C" {

size_t b200csr2csc_workspace_bytes(int64_t m, int64_t n, int64_t nnz) {
    if (!conv_dims_ok(m, n, nnz)) return 0;
    return rt_scratch_bytes(nnz);
}

int b200csr2csc(void* stream, int64_t m, int64_t n, int64_t nnz, const void* csr_val, const void* csr_row_ptr, const void* csr_col_ind,
                void* csc_val, void* csc_col_ptr, void* csc_row_ind, int value_bytes, int numeric, int32_t base, void* workspace,
                size_t workspace_bytes) {
    if (!conv_dims_ok(m, n, nnz) || (base != 0 && base != 1) || (nnz > 0 && (m == 0 || n == 0))) return -1;
    if (numeric && !width_ok(value_bytes)) return -1;
    if (!csc_col_ptr || !aligned(csc_col_ptr, 4)) return -1;
    if (nnz > 0) {
        if (!csr_row_ptr || !csr_col_ind || !csc_row_ind || !aligned(csr_row_ptr, 4) || !aligned(csr_col_ind, 4) || !aligned(csc_row_ind, 4))
            return -1;
        if (numeric && (!csr_val || !csc_val || !aligned(csr_val, value_bytes) || !aligned(csc_val, value_bytes))) return -1;
        if (!workspace || !aligned(workspace, 16) || workspace_bytes < rt_scratch_bytes(nnz)) return -1;
    }
    const cudaStream_t st = (cudaStream_t)stream;
    const int nz = (int)nnz;
    if (nz == 0) {
        rt_offsets(st, nullptr, 0, 0, n, base, (int*)csc_col_ptr);
        return (int)cudaGetLastError();
    }
    const int *sorted = nullptr, *perm = nullptr;
    rt_sort(st, (const int*)csr_col_ind, base, nullptr, nullptr, nz, n, rt_scratch((char*)workspace, nnz), nullptr, &sorted, &perm);
    rt_offsets(st, sorted, 0, nz, n, base, (int*)csc_col_ptr);
    rt_rows(st, (const int*)csr_row_ptr, base, m, perm, nz, base, (int*)csc_row_ind);
    if (numeric) rt_gather(st, value_bytes, csr_val, perm, nz, csc_val);
    return (int)cudaGetLastError();
}

size_t b200coosort_workspace_bytes(int64_t m, int64_t n, int64_t nnz) {
    if (!conv_dims_ok(m, n, nnz)) return 0;
    return rt_scratch_bytes(nnz) + round_up_256((size_t)nnz * 4);
}

int b200coosort(void* stream, int by_row, int64_t m, int64_t n, int64_t nnz, void* rows, void* cols, void* P, void* workspace,
                size_t workspace_bytes) {
    if (!conv_dims_ok(m, n, nnz)) return -1;
    if (nnz == 0) return 0;
    if (!rows || !cols || !P || !aligned(rows, 4) || !aligned(cols, 4) || !aligned(P, 4)) return -1;
    if (!workspace || !aligned(workspace, 16) || workspace_bytes < b200coosort_workspace_bytes(m, n, nnz)) return -1;
    const cudaStream_t st = (cudaStream_t)stream;
    const int nz = (int)nnz;
    int* first = (int*)(by_row ? rows : cols);
    int* second = (int*)(by_row ? cols : rows);
    const int64_t first_keys = (by_row ? m : n) + 1, second_keys = (by_row ? n : m) + 1;
    const RtScratch s = rt_scratch((char*)workspace, nnz);
    int* p1 = (int*)((char*)workspace + rt_scratch_bytes(nnz));
    // by the second key into p1, then stably by the first key read through p1: sigma, and the first keys in sorted order
    rt_sort(st, second, 0, nullptr, nullptr, nz, second_keys, s, p1, nullptr, nullptr);
    const int *first_sorted = nullptr, *sigma = nullptr;
    rt_sort(st, first, 0, p1, p1, nz, first_keys, s, nullptr, &first_sorted, &sigma);
    // the two buffers the last pass did not write are free: the second keys and P gathered by sigma, then all three copied home
    const int last = rt_passes(first_keys) - 1;
    int* second_sorted = s.k[(last + 1) & 1];
    int* p_sorted = s.v[(last + 1) & 1];
    rt_gather(st, 4, second, sigma, nz, second_sorted);
    rt_gather(st, 4, P, sigma, nz, p_sorted);
    const size_t b = (size_t)nnz * 4;
    cudaMemcpyAsync(first, first_sorted, b, cudaMemcpyDeviceToDevice, st);
    cudaMemcpyAsync(second, second_sorted, b, cudaMemcpyDeviceToDevice, st);
    cudaMemcpyAsync(P, p_sorted, b, cudaMemcpyDeviceToDevice, st);
    return (int)cudaGetLastError();
}

int b200coo2csr(void* stream, const void* coo_row_ind, int64_t nnz, int64_t m, void* csr_row_ptr, int32_t base) {
    if (!conv_dims_ok(m, 0, nnz) || (base != 0 && base != 1)) return -1;
    if (!csr_row_ptr || !aligned(csr_row_ptr, 4) || (nnz > 0 && (!coo_row_ind || !aligned(coo_row_ind, 4)))) return -1;
    rt_offsets((cudaStream_t)stream, (const int*)coo_row_ind, base, (int)nnz, m, base, (int*)csr_row_ptr);
    return (int)cudaGetLastError();
}

int b200csr2coo(void* stream, const void* csr_row_ptr, int64_t nnz, int64_t m, void* coo_row_ind, int32_t base) {
    if (!conv_dims_ok(m, 0, nnz) || (base != 0 && base != 1) || (nnz > 0 && m == 0)) return -1;
    if (nnz == 0) return 0;
    if (!csr_row_ptr || !coo_row_ind || !aligned(csr_row_ptr, 4) || !aligned(coo_row_ind, 4)) return -1;
    rt_rows((cudaStream_t)stream, (const int*)csr_row_ptr, base, m, nullptr, (int)nnz, base, (int*)coo_row_ind);
    return (int)cudaGetLastError();
}

int b200identity_permutation(void* stream, int64_t n, void* p) {
    if (n < 0 || n > INT32_MAX) return -1;
    if (n == 0) return 0;
    if (!p || !aligned(p, 4)) return -1;
    const unsigned grid = (unsigned)std::min<int64_t>((n + RT_THREADS - 1) / RT_THREADS, 65536);
    identity_permutation_kernel<<<grid, RT_THREADS, 0, (cudaStream_t)stream>>>((int*)p, (int)n);
    return (int)cudaGetLastError();
}

}  // extern "C"
