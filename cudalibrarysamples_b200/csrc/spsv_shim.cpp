// spsv_shim.cpp -- the cusparseSpSV_* symbols of libb200spsv.so (include/b200spsv.h).
//
// SpSV descriptors stay REAL cuSPARSE descriptors: _createDescr always creates one through the real library, so any call
// can still be forwarded, and a side table keyed by it remembers whether _analysis built our plan (and where).  Matrix
// and vector descriptors are read through the real getters, whoever created them, so this library works with or
// without libb200spmv.so in the process.
//
// Served natively: CSR, 32-bit indices, fp32 / fp64 with x, y and compute type of the same type, CUSPARSE_SPSV_ALG_DEFAULT,
// fill LOWER / UPPER, diag UNIT / NON_UNIT (read with cusparseSpMatGetAttribute), op NON_TRANSPOSE / TRANSPOSE, square A.
// Everything else is forwarded -- as is a NON_UNIT matrix in which analysis finds a row that stores no diagonal, and
// every call under B200SPMV_FORWARD=1.  B200SPMV_LOG=1 names the path of each call on stderr.
#include <cuda_runtime_api.h>
#include <cusparse.h>

#include <atomic>
#include <cstdio>
#include <cstdlib>
#include <mutex>
#include <unordered_map>

#include "../../include/b200spsv.h"
#include "real_cusparse.h"

namespace {

// Every real-library function this shim calls: expanded into the members of Real and into their loads.
#define SPSV_REAL_FNS(X)                                                                                                      \
    X(cusparseSpSV_createDescr) X(cusparseSpSV_destroyDescr) X(cusparseSpSV_bufferSize) X(cusparseSpSV_analysis)             \
    X(cusparseSpSV_solve) X(cusparseSpSV_updateMatrix) X(cusparseGetStream) X(cusparseGetPointerMode) X(cusparseSpMatGetFormat) \
    X(cusparseSpMatGetAttribute) X(cusparseConstCsrGet) X(cusparseConstDnVecGet)

struct Real {
    void* h = nullptr;
#define REAL_MEMBER(name) decltype(&::name) name = nullptr;
    SPSV_REAL_FNS(REAL_MEMBER)
#undef REAL_MEMBER
    bool forward = false, log = false;
};

Real*          g_real = nullptr;
std::once_flag g_once;

void init_real() {
    Real* r = new Real();
    r->forward = b200::env_flag("B200SPMV_FORWARD");
    r->log = b200::env_flag("B200SPMV_LOG");
    r->h = b200::open_real_cusparse("b200spsv");
#define REAL_LOAD(name) r->name = (decltype(r->name))b200::real_symbol(r->h, #name, "b200spsv");
    SPSV_REAL_FNS(REAL_LOAD)
#undef REAL_LOAD
    g_real = r;
}

inline Real& real() {
    std::call_once(g_once, init_real);
    return *g_real;
}

std::atomic<uint64_t> g_native{0}, g_forwarded{0}, g_analysis{0};

// What a natively analysed SpSV descriptor remembers: the plan's shape and workspace, and the updateMatrix overrides.
struct SvInfo {
    bool        native = false;
    void*       buffer = nullptr;
    int64_t     rows = 0, nnz = 0;
    int         op = 0, lower = 1, unit = 0;
    cudaDataType vtype = CUDA_R_32F;
    const void* values = nullptr;    // matA's values pointer at analysis, or cusparseSpSV_updateMatrix GENERAL's newValues
    const void* diag = nullptr;      // cusparseSpSV_updateMatrix DIAGONAL: rows values used instead of the stored diagonal
};

std::mutex                               g_mu;
std::unordered_map<const void*, SvInfo>  g_sv;

// The CSR matrix as the real library describes it, with its fill mode and diagonal type.
struct Csr {
    cusparseFormat_t    format = CUSPARSE_FORMAT_CSR;
    int64_t             rows = 0, cols = 0, nnz = 0;
    const void *        offsets = nullptr, *col_ind = nullptr, *values = nullptr;
    cusparseIndexType_t off_type = CUSPARSE_INDEX_32I, col_type = CUSPARSE_INDEX_32I;
    cusparseIndexBase_t base = CUSPARSE_INDEX_BASE_ZERO;
    cudaDataType        vtype = CUDA_R_32F;
    cusparseFillMode_t  fill = CUSPARSE_FILL_MODE_LOWER;
    cusparseDiagType_t  diag = CUSPARSE_DIAG_TYPE_NON_UNIT;
};

// false: not a descriptor the getters accept, or not CSR (both mean "forward")
bool get_csr(cusparseConstSpMatDescr_t d, Csr* m) {
    Real& R = real();
    if (!d || R.cusparseSpMatGetFormat(d, &m->format) != CUSPARSE_STATUS_SUCCESS || m->format != CUSPARSE_FORMAT_CSR) return false;
    if (R.cusparseConstCsrGet(d, &m->rows, &m->cols, &m->nnz, &m->offsets, &m->col_ind, &m->values, &m->off_type, &m->col_type,
                              &m->base, &m->vtype) != CUSPARSE_STATUS_SUCCESS)
        return false;
    if (R.cusparseSpMatGetAttribute(d, CUSPARSE_SPMAT_FILL_MODE, &m->fill, sizeof m->fill) != CUSPARSE_STATUS_SUCCESS ||
        R.cusparseSpMatGetAttribute(d, CUSPARSE_SPMAT_DIAG_TYPE, &m->diag, sizeof m->diag) != CUSPARSE_STATUS_SUCCESS)
        return false;
    return true;
}

bool get_vec(cusparseConstDnVecDescr_t d, int64_t* size, const void** values, cudaDataType* vtype) {
    return d && real().cusparseConstDnVecGet(d, size, values, vtype) == CUSPARSE_STATUS_SUCCESS;
}

// The call's shape, all read from descriptors; true when our kernel takes it.
bool native_shape(cusparseOperation_t op, cusparseConstSpMatDescr_t matA, cusparseConstDnVecDescr_t vecX, cusparseDnVecDescr_t vecY,
                  cudaDataType compute, cusparseSpSVAlg_t alg, Csr* m, int64_t* nx, const void** px, int64_t* ny, const void** py) {
    cudaDataType xt, yt;
    if (!get_csr(matA, m) || !get_vec(vecX, nx, px, &xt) || !get_vec(vecY, ny, py, &yt)) return false;
    if (!b200spsv_route((int)m->format, (int)op, (int)alg, (int)m->off_type, (int)m->col_type, (int)m->vtype, (int)xt, (int)yt,
                        (int)compute, (int)m->fill, (int)m->diag, m->rows, m->cols, m->nnz))
        return false;
    return *nx == m->rows && *ny == m->rows;
}

cusparseStatus_t to_status(int rc) {
    if (rc == 0) return CUSPARSE_STATUS_SUCCESS;
    if (rc == -1) return CUSPARSE_STATUS_INVALID_VALUE;
    return CUSPARSE_STATUS_EXECUTION_FAILED;
}

void note(const char* what) {
    if (real().log) fprintf(stderr, "[b200spsv] %s\n", what);
}

void set_entry(const void* d, const SvInfo& s) {
    std::lock_guard<std::mutex> lk(g_mu);
    g_sv[d] = s;
}

bool find_entry(const void* d, SvInfo* s) {
    std::lock_guard<std::mutex> lk(g_mu);
    auto it = g_sv.find(d);
    if (it == g_sv.end()) return false;
    *s = it->second;
    return true;
}

}  // namespace

extern "C" {

const char* b200spsv_version(void) { return "b200spsv 0.1 (sm_90a)"; }

int b200spsv_route(int format, int op, int alg, int off_type, int col_type, int a_vtype, int x_vtype, int y_vtype, int compute_type,
                   int fill, int diag, int64_t rows, int64_t cols, int64_t nnz) {
    if (format != CUSPARSE_FORMAT_CSR) return 0;                                       // COO, Sliced-ELL, ...
    if (op != CUSPARSE_OPERATION_NON_TRANSPOSE && op != CUSPARSE_OPERATION_TRANSPOSE) return 0;
    if (alg != CUSPARSE_SPSV_ALG_DEFAULT) return 0;
    if (off_type != CUSPARSE_INDEX_32I || col_type != CUSPARSE_INDEX_32I) return 0;
    if (a_vtype != CUDA_R_32F && a_vtype != CUDA_R_64F) return 0;                      // complex, 16-bit, integer
    if (x_vtype != a_vtype || y_vtype != a_vtype || compute_type != a_vtype) return 0; // mixed types
    if ((fill != CUSPARSE_FILL_MODE_LOWER && fill != CUSPARSE_FILL_MODE_UPPER) ||
        (diag != CUSPARSE_DIAG_TYPE_NON_UNIT && diag != CUSPARSE_DIAG_TYPE_UNIT))
        return 0;
    if (rows != cols || rows < 0 || rows >= INT32_MAX || nnz < 0 || nnz >= INT32_MAX) return 0;   // the real library's verdict
    return 1;
}

void b200spsv_get_stats(uint64_t* native_calls, uint64_t* forwarded_calls, uint64_t* analysis_calls) {
    if (native_calls) *native_calls = g_native.load();
    if (forwarded_calls) *forwarded_calls = g_forwarded.load();
    if (analysis_calls) *analysis_calls = g_analysis.load();
}

void b200spsv_reset_stats(void) {
    g_native = 0;
    g_forwarded = 0;
    g_analysis = 0;
}

cusparseStatus_t cusparseSpSV_createDescr(cusparseSpSVDescr_t* descr) {
    cusparseStatus_t st = real().cusparseSpSV_createDescr(descr);
    if (st == CUSPARSE_STATUS_SUCCESS) set_entry((const void*)*descr, SvInfo());
    return st;
}

cusparseStatus_t cusparseSpSV_destroyDescr(cusparseSpSVDescr_t descr) {
    {
        std::lock_guard<std::mutex> lk(g_mu);
        g_sv.erase((const void*)descr);
    }
    return real().cusparseSpSV_destroyDescr(descr);
}

cusparseStatus_t cusparseSpSV_bufferSize(cusparseHandle_t handle, cusparseOperation_t opA, const void* alpha,
                                         cusparseConstSpMatDescr_t matA, cusparseConstDnVecDescr_t vecX, cusparseDnVecDescr_t vecY,
                                         cudaDataType computeType, cusparseSpSVAlg_t alg, cusparseSpSVDescr_t spsvDescr,
                                         size_t* bufferSize) {
    // The real size always: a forward decided only at analysis then runs the real analysis in the same buffer.
    Real& R = real();
    cusparseStatus_t st = R.cusparseSpSV_bufferSize(handle, opA, alpha, matA, vecX, vecY, computeType, alg, spsvDescr, bufferSize);
    if (st != CUSPARSE_STATUS_SUCCESS || R.forward || !bufferSize) return st;
    Csr m; int64_t nx, ny; const void *px, *py;
    if (native_shape(opA, matA, vecX, vecY, computeType, alg, &m, &nx, &px, &ny, &py)) {
        const size_t ours = b200spsv_csr_workspace_bytes(m.rows, m.nnz, opA != CUSPARSE_OPERATION_NON_TRANSPOSE);
        if (ours > *bufferSize) *bufferSize = ours;
    }
    return st;
}

cusparseStatus_t cusparseSpSV_analysis(cusparseHandle_t handle, cusparseOperation_t opA, const void* alpha,
                                       cusparseConstSpMatDescr_t matA, cusparseConstDnVecDescr_t vecX, cusparseDnVecDescr_t vecY,
                                       cudaDataType computeType, cusparseSpSVAlg_t alg, cusparseSpSVDescr_t spsvDescr,
                                       void* externalBuffer) {
    Real& R = real();
    auto forward = [&](const char* why) {
        if (R.log) fprintf(stderr, "[b200spsv] analysis forwarded to libcusparse (%s)\n", why);
        g_forwarded++;
        SvInfo s;
        set_entry((const void*)spsvDescr, s);
        return R.cusparseSpSV_analysis(handle, opA, alpha, matA, vecX, vecY, computeType, alg, spsvDescr, externalBuffer);
    };
    if (R.forward) return forward("B200SPMV_FORWARD");
    SvInfo s;
    if (!handle || !spsvDescr || !find_entry((const void*)spsvDescr, &s)) return forward("descriptor not created here");
    Csr m; int64_t nx, ny; const void *px, *py;
    if (!native_shape(opA, matA, vecX, vecY, computeType, alg, &m, &nx, &px, &ny, &py)) return forward("unsupported combination");
    // The closed library takes a NULL buffer at face value and its analysis kernels fault writing through it: refuse it.
    if (!externalBuffer) return CUSPARSE_STATUS_INVALID_VALUE;
    if ((uintptr_t)externalBuffer & 15) return forward("misaligned externalBuffer");
    cudaStream_t stream = nullptr;
    cusparseStatus_t st = R.cusparseGetStream(handle, &stream);
    if (st != CUSPARSE_STATUS_SUCCESS) return st;
    cudaStreamCaptureStatus cap = cudaStreamCaptureStatusNone;
    if (cudaStreamIsCapturing(stream, &cap) != cudaSuccess || cap != cudaStreamCaptureStatusNone)
        return forward("stream is being captured: the missing-diagonal check cannot read back");
    const int lower = m.fill == CUSPARSE_FILL_MODE_LOWER, unit = m.diag == CUSPARSE_DIAG_TYPE_UNIT;
    const int tr = opA != CUSPARSE_OPERATION_NON_TRANSPOSE;
    int64_t missing = 0;
    const int rc = b200spsv_csr_analysis((void*)stream, m.rows, m.nnz, m.offsets, m.col_ind, (int32_t)m.base, lower, unit, tr,
                                         externalBuffer, &missing);
    if (rc != 0) return to_status(rc);
    if (!unit && missing > 0) return forward("NON_UNIT matrix with a row that stores no diagonal");
    s.native = true;
    s.buffer = externalBuffer;
    s.rows = m.rows;
    s.nnz = m.nnz;
    s.op = tr;
    s.lower = lower;
    s.unit = unit;
    s.vtype = m.vtype;
    s.values = m.values;
    s.diag = nullptr;
    set_entry((const void*)spsvDescr, s);
    g_analysis++;
    if (R.log)
        fprintf(stderr, "[b200spsv] analysis native rows=%lld nnz=%lld %s %s%s base=%d\n", (long long)m.rows, (long long)m.nnz,
                lower ? "lower" : "upper", unit ? "unit" : "non-unit", tr ? " transposed" : "", (int)m.base);
    return CUSPARSE_STATUS_SUCCESS;
}

cusparseStatus_t cusparseSpSV_solve(cusparseHandle_t handle, cusparseOperation_t opA, const void* alpha, cusparseConstSpMatDescr_t matA,
                                    cusparseConstDnVecDescr_t vecX, cusparseDnVecDescr_t vecY, cudaDataType computeType,
                                    cusparseSpSVAlg_t alg, cusparseSpSVDescr_t spsvDescr) {
    Real& R = real();
    SvInfo s;
    if (R.forward || !spsvDescr || !find_entry((const void*)spsvDescr, &s) || !s.native) {
        note("solve forwarded to libcusparse (descriptor analysed by the closed library)");
        g_forwarded++;
        return R.cusparseSpSV_solve(handle, opA, alpha, matA, vecX, vecY, computeType, alg, spsvDescr);
    }
    if (!handle || !alpha) return CUSPARSE_STATUS_INVALID_VALUE;
    Csr m; int64_t nx, ny; const void *px, *py;
    if (!native_shape(opA, matA, vecX, vecY, computeType, alg, &m, &nx, &px, &ny, &py) || m.rows != s.rows || m.nnz != s.nnz ||
        m.vtype != s.vtype || (int)(opA != CUSPARSE_OPERATION_NON_TRANSPOSE) != s.op)
        return CUSPARSE_STATUS_INVALID_VALUE;      // not the call this descriptor was analysed for
    cudaStream_t stream = nullptr;
    cusparseStatus_t st = R.cusparseGetStream(handle, &stream);
    if (st != CUSPARSE_STATUS_SUCCESS) return st;
    cusparsePointerMode_t pm = CUSPARSE_POINTER_MODE_HOST;
    st = R.cusparseGetPointerMode(handle, &pm);
    if (st != CUSPARSE_STATUS_SUCCESS) return st;
    if (R.log)
        fprintf(stderr, "[b200spsv] solve native rows=%lld nnz=%lld%s\n", (long long)m.rows, (long long)m.nnz,
                s.diag ? " (updated diagonal)" : "");
    // The values pointer is the one analysis saw (as in the closed library: a later cusparseSpMatSetValues does not reach
    // an analysed solve; cusparseSpSV_updateMatrix does).  Its contents are read now.
    const int rc = b200spsv_csr_solve((void*)stream, m.vtype == CUDA_R_64F, m.rows, m.nnz, s.lower, s.unit, s.op, s.values, s.diag,
                                      alpha, pm == CUSPARSE_POINTER_MODE_DEVICE, px, (void*)py, s.buffer);
    g_native++;
    return to_status(rc);
}

// GENERAL: the solve uses newValues in place of the values analysis saw (and the stored diagonal again).  DIAGONAL: newValues holds
// rows diagonal values that replace the stored ones.  Both only change what the next solve reads: the plan is structure.
cusparseStatus_t cusparseSpSV_updateMatrix(cusparseHandle_t handle, cusparseSpSVDescr_t spsvDescr, void* newValues,
                                           cusparseSpSVUpdate_t updatePart) {
    Real& R = real();
    SvInfo s;
    if (R.forward || !spsvDescr || !find_entry((const void*)spsvDescr, &s) || !s.native) {
        note("updateMatrix forwarded to libcusparse");
        g_forwarded++;
        return R.cusparseSpSV_updateMatrix(handle, spsvDescr, newValues, updatePart);
    }
    if (!handle || (!newValues && s.rows > 0)) return CUSPARSE_STATUS_INVALID_VALUE;
    if (updatePart == CUSPARSE_SPSV_UPDATE_GENERAL) {
        s.values = newValues;
        s.diag = nullptr;
    } else if (updatePart == CUSPARSE_SPSV_UPDATE_DIAGONAL) {
        s.diag = newValues;
    } else {
        return CUSPARSE_STATUS_INVALID_VALUE;
    }
    set_entry((const void*)spsvDescr, s);
    note(updatePart == CUSPARSE_SPSV_UPDATE_GENERAL ? "updateMatrix native (values)" : "updateMatrix native (diagonal)");
    return CUSPARSE_STATUS_SUCCESS;
}

}  // extern "C"
