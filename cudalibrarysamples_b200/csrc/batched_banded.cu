// batched_banded.cu -- batched penta- and tridiagonal solves in the interleaved layout (cusparse<t>gpsvInterleavedBatch,
// cusparse<t>gtsvInterleavedBatch) on H100 (sm_90a): the launches of batched_banded.cuh's kernels.  DESIGN.md 3.25.
#include "batched_banded.cuh"
#include "../../include/b200spmv.h"

#include <cuda_runtime.h>

namespace b200 {
namespace {

// bytes of one value of a cudaDataType the solves take; 0 for any other
size_t band_value_bytes(int vtype) {
    switch (vtype) {
    case CUDA_R_32F: return 4;
    case CUDA_R_64F: case CUDA_C_32F: return 8;
    case CUDA_C_64F: return 16;
    default: return 0;
    }
}

bool aligned(const void* p, size_t a) { return ((uintptr_t)p & (a - 1)) == 0; }

// systems up to INT32_MAX rows and as many systems: every element index m * batch fits an int64_t many times over
bool band_dims_ok(int64_t m, int64_t batch) { return m >= 1 && batch >= 1 && m <= INT32_MAX && batch <= INT32_MAX; }

template <typename V, int P, int METHOD>
int launch(cudaStream_t st, const void* const* diag, void* x, int64_t m, int64_t batch, void* work) {
    BandArgs<V> a{};
    for (int o = 0; o <= 2 * P; o++) a.diag[o] = (const V*)diag[o];
    a.x = (V*)x;
    a.work = (V*)work;
    a.m = m;
    a.batch = batch;
    banded_interleaved_kernel<V, P, METHOD><<<(unsigned)((batch + BAND_BLOCK - 1) / BAND_BLOCK), BAND_BLOCK, 0, st>>>(a);
    return (int)cudaGetLastError();
}

template <int P, int METHOD>
int dispatch(void* stream, int vtype, const void* const* diag, void* x, int64_t m, int64_t batch, void* work) {
    const cudaStream_t st = (cudaStream_t)stream;
    switch (vtype) {
    case CUDA_R_32F: return launch<float, P, METHOD>(st, diag, x, m, batch, work);
    case CUDA_R_64F: return launch<double, P, METHOD>(st, diag, x, m, batch, work);
    case CUDA_C_32F: return launch<cplx<float>, P, METHOD>(st, diag, x, m, batch, work);
    case CUDA_C_64F: return launch<cplx<double>, P, METHOD>(st, diag, x, m, batch, work);
    default: return -1;
    }
}

// NULL or misaligned operands, a workspace too small: -1 before anything is launched
bool operands_ok(int vtype, const void* const* diag, int n, const void* x, const void* work, int64_t m, int64_t batch, size_t need) {
    const size_t w = band_value_bytes(vtype);
    if (!w || !band_dims_ok(m, batch) || !x || !aligned(x, w) || !work || !aligned(work, 16) || need == 0) return false;
    for (int o = 0; o < n; o++)
        if (!diag[o] || !aligned(diag[o], w)) return false;
    return true;
}

size_t work_bytes(int vtype, int W, int64_t m, int64_t batch) {
    if (!band_value_bytes(vtype) || !band_dims_ok(m, batch)) return 0;
    return (size_t)W * (size_t)m * (size_t)batch * band_value_bytes(vtype);
}

}  // namespace
}  // namespace b200

using namespace b200;

extern "C" {

size_t b200gpsv_interleaved_workspace_bytes(int vtype, int64_t m, int64_t batch) {
    return work_bytes(vtype, band_width<2, BAND_GIVENS>::W, m, batch);
}

size_t b200gtsv_interleaved_workspace_bytes(int vtype, int algo, int64_t m, int64_t batch) {
    switch (algo) {
    case 0: return work_bytes(vtype, band_width<1, BAND_THOMAS>::W, m, batch);
    case 1: return work_bytes(vtype, band_width<1, BAND_PIVOT_LU>::W, m, batch);
    case 2: return work_bytes(vtype, band_width<1, BAND_GIVENS>::W, m, batch);
    default: return 0;
    }
}

int b200gpsv_interleaved(void* stream, int vtype, int64_t m, const void* ds, const void* dl, const void* d, const void* du,
                         const void* dw, void* x, int64_t batch, void* workspace) {
    const void* diag[5] = {ds, dl, d, du, dw};
    if (!operands_ok(vtype, diag, 5, x, workspace, m, batch, b200gpsv_interleaved_workspace_bytes(vtype, m, batch))) return -1;
    return dispatch<2, BAND_GIVENS>(stream, vtype, diag, x, m, batch, workspace);
}

int b200gtsv_interleaved(void* stream, int vtype, int algo, int64_t m, const void* dl, const void* d, const void* du, void* x,
                         int64_t batch, void* workspace) {
    const void* diag[3] = {dl, d, du};
    if (!operands_ok(vtype, diag, 3, x, workspace, m, batch, b200gtsv_interleaved_workspace_bytes(vtype, algo, m, batch))) return -1;
    switch (algo) {
    case 0: return dispatch<1, BAND_THOMAS>(stream, vtype, diag, x, m, batch, workspace);
    case 1: return dispatch<1, BAND_PIVOT_LU>(stream, vtype, diag, x, m, batch, workspace);
    default: return dispatch<1, BAND_GIVENS>(stream, vtype, diag, x, m, batch, workspace);
    }
}

}  // extern "C"
