// emulate_banded.cpp -- TEST INFRASTRUCTURE: the kernels of cudalibrarysamples_b200/csrc/batched_banded.cuh, THE SAME SOURCE,
// compiled for the host on top of cuda_emulation.h and exported for tests/test_banded_cpu.py (ctypes).  The launch geometry is the
// device one (BAND_BLOCK threads per CTA, one thread per system); the batch count need not fill the last CTA.
#define B200_HOST_EMULATION
#include "cuda_emulation.h"
#include "batched_banded.cuh"

using namespace b200;

namespace {

template <typename V, int P, int METHOD>
int run(const void* const* diag, void* x, long long m, long long batch, void* work) {
    BandArgs<V> a{};
    for (int o = 0; o <= 2 * P; o++) a.diag[o] = (const V*)diag[o];
    a.x = (V*)x;
    a.work = (V*)work;
    a.m = m;
    a.batch = batch;
    emu::launch((unsigned)((batch + BAND_BLOCK - 1) / BAND_BLOCK), BAND_BLOCK, [&] { banded_interleaved_kernel<V, P, METHOD>(a); });
    return 0;
}

// vtype: 0 float, 1 double, 2 complex float, 3 complex double
template <int P, int METHOD>
int by_type(int vtype, const void* const* diag, void* x, long long m, long long batch, void* work) {
    switch (vtype) {
    case 0: return run<float, P, METHOD>(diag, x, m, batch, work);
    case 1: return run<double, P, METHOD>(diag, x, m, batch, work);
    case 2: return run<cplx<float>, P, METHOD>(diag, x, m, batch, work);
    case 3: return run<cplx<double>, P, METHOD>(diag, x, m, batch, work);
    default: return -1;
    }
}

}  // namespace

extern "C" {

// method: 0 gpsv (Givens, P = 2); 1, 2, 3: gtsv algo 0 (Thomas), 1 (pivoted LU), 2 (Givens); work: W * m * batch values
int emu_banded(int method, int vtype, long long m, long long batch, const void* ds, const void* dl, const void* d, const void* du,
               const void* dw, void* x, void* work) {
    const void* penta[5] = {ds, dl, d, du, dw};
    const void* tri[3] = {dl, d, du};
    switch (method) {
    case 0: return by_type<2, BAND_GIVENS>(vtype, penta, x, m, batch, work);
    case 1: return by_type<1, BAND_THOMAS>(vtype, tri, x, m, batch, work);
    case 2: return by_type<1, BAND_PIVOT_LU>(vtype, tri, x, m, batch, work);
    case 3: return by_type<1, BAND_GIVENS>(vtype, tri, x, m, batch, work);
    default: return -1;
    }
}

}  // extern "C"
