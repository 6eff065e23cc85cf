// spmv_generic.cu -- the rest of cusparseSpMV's real-valued argument space on H100 (sm_90a), SURVEY.md 8(f)-3:
//   * 64-bit indices: CSR row offsets / column indices (64/64 and 64/32), COO indices, Sliced-ELL offsets / columns;
//   * mixed precision: A in fp32 with x, y and the arithmetic in fp64 (the closed library's
//     csrmv_v3_kernel<..., float, double, double, double>);
//   * opA = TRANSPOSE for the combinations above and for Sliced-ELL of any index width;
//   * CSR calls that arrive without a usable externalBuffer (the tile / flat kernels need their plan in it).
// Rounds 1-2 handed all of these to the closed library.  The 32-bit, single-type cases keep their specialised kernels
// (spmv_csr*.cu, spmv_coo_sell.cu); what lands here is the long tail, served by deliberately plain kernels:
//
//   csr_generic_kernel            L = 4..32 lanes per row (chosen from nnz / rows), lanes stride through the row, one shuffle
//                                 tree per row; a warp owns 32 / L consecutive rows per trip of a warp-uniform loop;
//   csr_generic_transpose_kernel  the same walk, one RED.ADD per non-zero into y[col] (y pre-scaled by beta);
//   coo_generic_kernel            one RED.ADD per entry (y pre-scaled by beta): any order of the entries; A^T = the same
//                                 kernel with the two index arrays swapped by the caller;
//   sell_generic_kernel           one thread per row, slice-column-major walk, padding (column -1 + base) skipped;
//   sell_generic_transpose_kernel the same walk, one RED.ADD per entry.
//
// All index arithmetic is 64-bit, no workspace, no plan, no host synchronisation (CUDA-graph capturable).  Kernels that use
// atomics (transposes, COO) agree with the oracle to tolerance, not bit for bit; the others sum a row in a fixed order.
// Call sites these serve: cusparseCreateCsr(..., CUSPARSE_INDEX_64I, ...) / cusparseCreateCoo / cusparseCreateSlicedEll
// (cusparse.h:5208, 5362, 5470; index types :5002-5007) followed by the SpMV trio (cusparse.h:5679-5712).
#include "spmv_generic_kernels.cuh"
#include "config.h"
#include "../../include/b200spmv.h"

namespace b200 {

// ------------------------------------------------------------------------------------------------ host side
static unsigned grid_for(long long threads) {
    long long ctas = (threads + GEN_BLOCK - 1) / GEN_BLOCK;
    if (ctas < 1) ctas = 1;
    if (ctas > GEN_MAX_CTAS) ctas = GEN_MAX_CTAS;
    return (unsigned)ctas;
}

// y = beta * y ahead of a kernel that only adds (skipped when beta is known to be 1 on the host)
template <typename XT>
static int prescale(cudaStream_t stream, XT* y, long long n, const Scalars<XT>& s, int on_device) {
    if (n <= 0 || (!on_device && s.beta == XT(1))) return 0;
    gen_scale_y_kernel<XT><<<grid_for(n), GEN_BLOCK, 0, stream>>>(y, n, s);
    return (int)cudaGetLastError();
}

struct GenCall {
    cudaStream_t stream;
    int          transpose, on_device;
    long long    rows, cols, nnz, base, slice_size;
    const void * off, *col, *val, *alpha, *beta, *x;
    void*        y;
};

template <typename OffT, typename ColT, typename AT, typename XT>
static GenArgs<OffT, ColT, AT, XT> make_args(const GenCall& c) {
    GenArgs<OffT, ColT, AT, XT> a;
    a.off = (const OffT*)c.off; a.col = (const ColT*)c.col; a.val = (const AT*)c.val; a.x = (const XT*)c.x; a.y = (XT*)c.y;
    a.rows = c.rows; a.cols = c.cols; a.nnz = c.nnz; a.base = c.base; a.slice_size = c.slice_size;
    set_scalars<XT>(a.s, c.alpha, c.beta, c.on_device);
    return a;
}

template <typename OffT, typename ColT, typename AT, typename XT>
static int launch_csr_generic(const GenCall& c) {
    auto a = make_args<OffT, ColT, AT, XT>(c);
    const long long mean = c.rows > 0 ? c.nnz / c.rows : 0;
    const int lanes_log2 = mean <= 4 ? 2 : mean <= 8 ? 3 : mean <= 16 ? 4 : 5;
    const unsigned grid = grid_for(c.rows << lanes_log2);
    if (c.transpose) {
        stats().last_csr_kernel = "b200::csr_generic_transpose_kernel";
        const int e = prescale<XT>(c.stream, a.y, c.cols, a.s, c.on_device);
        if (e != 0 || c.rows == 0 || c.nnz == 0) return e;
        csr_generic_transpose_kernel<OffT, ColT, AT, XT><<<grid, GEN_BLOCK, 0, c.stream>>>(a, lanes_log2);
        return (int)cudaGetLastError();
    }
    if (c.rows == 0) return 0;
    stats().last_csr_kernel = "b200::csr_generic_kernel";
    csr_generic_kernel<OffT, ColT, AT, XT><<<grid, GEN_BLOCK, 0, c.stream>>>(a, lanes_log2);
    return (int)cudaGetLastError();
}

template <typename OffT, typename ColT, typename AT, typename XT>
static int launch_coo_generic(const GenCall& c) {
    auto a = make_args<OffT, ColT, AT, XT>(c);
    const int e = prescale<XT>(c.stream, a.y, c.rows, a.s, c.on_device);
    if (e != 0 || c.nnz == 0 || c.rows == 0) return e;
    coo_generic_kernel<OffT, ColT, AT, XT><<<grid_for(c.nnz), GEN_BLOCK, 0, c.stream>>>(a);
    return (int)cudaGetLastError();
}

template <typename OffT, typename ColT, typename AT, typename XT>
static int launch_sell_generic(const GenCall& c) {
    auto a = make_args<OffT, ColT, AT, XT>(c);
    if (c.transpose) {
        const int e = prescale<XT>(c.stream, a.y, c.cols, a.s, c.on_device);
        if (e != 0 || c.rows == 0) return e;
        sell_generic_kernel<OffT, ColT, AT, XT, true><<<grid_for(c.rows), GEN_BLOCK, 0, c.stream>>>(a);
        return (int)cudaGetLastError();
    }
    if (c.rows == 0) return 0;
    sell_generic_kernel<OffT, ColT, AT, XT, false><<<grid_for(c.rows), GEN_BLOCK, 0, c.stream>>>(a);
    return (int)cudaGetLastError();
}

// (offsets 64-bit?, columns 64-bit?, A fp64?, x / y fp64?) -> one instantiation; 32-bit offsets with 64-bit columns and
// fp64 A with fp32 x / y are not combinations the closed library takes either
#define B200_GEN_DISPATCH(FN, off64, col64, a_dtype, xy_dtype, call)                                               \
    switch (((off64) ? 8 : 0) | ((col64) ? 4 : 0) | ((a_dtype) ? 2 : 0) | ((xy_dtype) ? 1 : 0)) {                   \
        case 0:  return FN<int32_t, int32_t, float, float>(call);                                                   \
        case 1:  return FN<int32_t, int32_t, float, double>(call);                                                  \
        case 3:  return FN<int32_t, int32_t, double, double>(call);                                                 \
        case 8:  return FN<int64_t, int32_t, float, float>(call);                                                   \
        case 9:  return FN<int64_t, int32_t, float, double>(call);                                                  \
        case 11: return FN<int64_t, int32_t, double, double>(call);                                                 \
        case 12: return FN<int64_t, int64_t, float, float>(call);                                                   \
        case 13: return FN<int64_t, int64_t, float, double>(call);                                                  \
        case 15: return FN<int64_t, int64_t, double, double>(call);                                                 \
        default: return -1;                                                                                         \
    }

}  // namespace b200

using namespace b200;

static bool gen_types_ok(int a_dtype, int xy_dtype) {
    return (a_dtype == 0 || a_dtype == 1) && (xy_dtype == 0 || xy_dtype == 1) && a_dtype <= xy_dtype;
}

extern "C" {

int b200spmv_csr_generic_mv(void* stream, int off64, int col64, int a_dtype, int xy_dtype, int transpose, int64_t rows, int64_t cols,
                            int64_t nnz, const void* row_offsets, const void* col_ind, const void* values, int64_t base,
                            const void* alpha, const void* beta, int scalars_on_device, const void* x, void* y) {
    if (rows < 0 || cols < 0 || nnz < 0 || !alpha || !beta || !gen_types_ok(a_dtype, xy_dtype)) return -1;
    const int64_t ny = transpose ? cols : rows;
    if (ny == 0) return 0;
    if (!y || (rows > 0 && !row_offsets) || (nnz > 0 && (!col_ind || !values || !x))) return -1;
    GenCall c{(cudaStream_t)stream, transpose, scalars_on_device, rows, cols, nnz, base, 0, row_offsets, col_ind, values, alpha, beta, x, y};
    B200_GEN_DISPATCH(launch_csr_generic, off64, col64, a_dtype, xy_dtype, c)
}

int b200spmv_coo_generic_mv(void* stream, int idx64, int a_dtype, int xy_dtype, int64_t rows, int64_t cols, int64_t nnz,
                            const void* row_ind, const void* col_ind, const void* values, int64_t base, const void* alpha,
                            const void* beta, int scalars_on_device, const void* x, void* y) {
    if (rows < 0 || cols < 0 || nnz < 0 || !alpha || !beta || !gen_types_ok(a_dtype, xy_dtype)) return -1;
    if (rows == 0) return 0;
    if (!y || (nnz > 0 && (!row_ind || !col_ind || !values || !x))) return -1;
    GenCall c{(cudaStream_t)stream, 0, scalars_on_device, rows, cols, nnz, base, 0, row_ind, col_ind, values, alpha, beta, x, y};
    B200_GEN_DISPATCH(launch_coo_generic, idx64, idx64, a_dtype, xy_dtype, c)
}

int b200spmv_sell_generic_mv(void* stream, int off64, int col64, int a_dtype, int xy_dtype, int transpose, int64_t rows, int64_t cols,
                             int64_t slice_size, const void* slice_offsets, const void* col_ind, const void* values, int64_t base,
                             const void* alpha, const void* beta, int scalars_on_device, const void* x, void* y) {
    if (rows < 0 || cols < 0 || slice_size <= 0 || !alpha || !beta || !gen_types_ok(a_dtype, xy_dtype)) return -1;
    const int64_t ny = transpose ? cols : rows;
    if (ny == 0) return 0;
    if (!y || (rows > 0 && !slice_offsets)) return -1;
    GenCall c{(cudaStream_t)stream, transpose, scalars_on_device, rows, cols, 0, base, slice_size, slice_offsets, col_ind, values, alpha, beta, x, y};
    B200_GEN_DISPATCH(launch_sell_generic, off64, col64, a_dtype, xy_dtype, c)
}

}  // extern "C"
