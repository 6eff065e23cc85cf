// bicgstab_fused.cu -- the BLAS-1 part of an unpreconditioned BiCGStab iteration (the loop of
// cuSPARSE/bicgstab/bicgstab_example.c:212-351 with M = I), fused, with every scalar and every decision on the device.
//
// One iteration around the two products v = A p and t = A s (18 whole-vector passes, b200cg_dot's 2 included):
//     b200cg_dot            denom = r0 . v                                                            (2 passes)
//     b200bicgstab_update_s alpha = rho_new / denom;  s = r - alpha v;  s2 = s . s                     (3)
//     b200bicgstab_dot2     ts = t . s,  tt = t . t                                                   (2)
//     b200bicgstab_update_xr omega = ts / tt;  x += alpha p + omega s;  r = s - omega t;
//                           rho_new = r0 . r,  r2 = r . r                                             (7)
//     b200bicgstab_update_p beta = (rho_new / rho) (alpha / omega);  p = r + beta (p - omega v)          (4)
//
// The state block (include/b200spmv.h) holds the scalars, a status word, the iteration counter and the residual history.
// Decisions (convergence, breakdown) are taken at kernel entry from reduced scalars only, which a multi-GPU caller
// all-reduces in between, so every rank takes the same decision at the same iteration.  Once the status leaves RUNNING,
// every kernel of this file returns at entry: x, r, p and the state stay bit-identical however many iterations a CUDA graph
// replays past the decision.
//
// No kernel writes a slot that its own CTAs read.  A transition that also updates vectors (converged at s) publishes the
// status from the CTA that arrives last in the reduction, after every CTA has read it; the other transitions update no
// vector, so a CTA that already sees the new status does the same work (none) as one that does not.  That is why
// rho <- rho_new happens in update_s (which reads rho_new only), not in update_p (which reads rho).
#include <cuda_runtime.h>
#include <stdint.h>
#include <math.h>
#include "cg_reduce.cuh"
#include "../../include/b200spmv.h"

namespace b200bicgstab {

using namespace b200cg;

constexpr int HEADER_BYTES = 96;            // 10 scalar slots, status, iterations, history capacity, padding
constexpr int STATUS_BYTE = 80, ITER_BYTE = 84, CAP_BYTE = 88;

struct State {
    double* s;
    __device__ explicit State(double* p) : s(p) {}
    __device__ int& status() const { return *reinterpret_cast<int*>(reinterpret_cast<char*>(s) + STATUS_BYTE); }
    __device__ int& iters() const { return *reinterpret_cast<int*>(reinterpret_cast<char*>(s) + ITER_BYTE); }
    __device__ int cap() const { return *reinterpret_cast<const int*>(reinterpret_cast<const char*>(s) + CAP_BYTE); }
    __device__ double* history() const { return reinterpret_cast<double*>(reinterpret_cast<char*>(s) + HEADER_BYTES); }
    // counts a finished iteration and records ||r|| after it
    __device__ void finish_iteration(double r2) const {
        const int k = ++iters();
        if (k < cap()) history()[k] = sqrt(r2);
    }
};

__device__ __forceinline__ bool below(double sq, double threshold) { return sqrt(sq) < threshold; }

// r = p = r0; rho = rho_new (= r0 . r0, already reduced); threshold; status; counter; history[0]
__global__ void __launch_bounds__(BLOCK) init_kernel(int64_t n, const double* __restrict__ r0, double* __restrict__ r,
                                                     double* __restrict__ p, double* __restrict__ state, int32_t cap, double tol) {
    const int64_t stride = (int64_t)gridDim.x * BLOCK * 2;
    for (int64_t i = ((int64_t)blockIdx.x * BLOCK + threadIdx.x) * 2; i < n; i += stride) {
        if (i + 1 < n) {
            const double2 v = *reinterpret_cast<const double2*>(r0 + i);
            *reinterpret_cast<double2*>(r + i) = v;
            *reinterpret_cast<double2*>(p + i) = v;
        } else {
            r[i] = r0[i];
            p[i] = r0[i];
        }
    }
    if (blockIdx.x == 0 && threadIdx.x == 0) {
        const State st(state);
        const double rho = state[B200BICGSTAB_RHO_NEW], nrm = sqrt(rho);
        state[B200BICGSTAB_RHO] = rho;
        state[B200BICGSTAB_R2] = rho;
        state[B200BICGSTAB_THRESHOLD] = tol < 0 ? -1.0 : tol * nrm;
        *reinterpret_cast<int*>(reinterpret_cast<char*>(state) + CAP_BYTE) = cap;
        st.iters() = 0;
        st.status() = !isfinite(rho) ? B200BICGSTAB_BREAKDOWN_NONFINITE : rho == 0 ? B200BICGSTAB_CONVERGED_R : B200BICGSTAB_RUNNING;
        if (cap > 0) st.history()[0] = nrm;
    }
}

// alpha = rho_new / denom;  s = r - alpha v;  s2 = s . s;  the last CTA publishes alpha and rho <- rho_new
__global__ void __launch_bounds__(BLOCK) update_s_kernel(int64_t n, const double* __restrict__ r, const double* __restrict__ v,
                                                         double* __restrict__ s, double* __restrict__ state, double* __restrict__ ws) {
    __shared__ double sred[BLOCK / 32];
    const State st(state);
    if (st.status() != B200BICGSTAB_RUNNING) return;
    const double denom = state[B200BICGSTAB_DENOM], alpha = state[B200BICGSTAB_RHO_NEW] / denom;
    const int next = denom == 0 ? B200BICGSTAB_BREAKDOWN_DENOM : !isfinite(alpha) ? B200BICGSTAB_BREAKDOWN_NONFINITE : B200BICGSTAB_RUNNING;
    if (next != B200BICGSTAB_RUNNING) {
        if (blockIdx.x == 0 && threadIdx.x == 0) st.status() = next;
        return;
    }
    double acc = 0;
    const int64_t stride = (int64_t)gridDim.x * BLOCK * 2;
    for (int64_t i = ((int64_t)blockIdx.x * BLOCK + threadIdx.x) * 2; i < n; i += stride) {
        if (i + 1 < n) {
            const double2 rr = *reinterpret_cast<const double2*>(r + i), vv = *reinterpret_cast<const double2*>(v + i);
            double2 ss;
            ss.x = rr.x - alpha * vv.x; ss.y = rr.y - alpha * vv.y;
            *reinterpret_cast<double2*>(s + i) = ss;
            acc += ss.x * ss.x + ss.y * ss.y;
        } else {
            const double sn = r[i] - alpha * v[i];
            s[i] = sn;
            acc += sn * sn;
        }
    }
    double part[1] = {acc};
    block_sum_k<1>(part, sred);
    if (threadIdx.x == 0 && grid_sum_finish_k<1>(part, ws, state + B200BICGSTAB_S2)) {
        state[B200BICGSTAB_ALPHA] = alpha;
        state[B200BICGSTAB_RHO] = state[B200BICGSTAB_RHO_NEW];
    }
}

// ts = t . s and tt = t . t in one pass
__global__ void __launch_bounds__(BLOCK) dot2_kernel(int64_t n, const double* __restrict__ t, const double* __restrict__ s,
                                                     double* __restrict__ state, double* __restrict__ ws) {
    __shared__ double sred[2 * (BLOCK / 32)];
    if (State(state).status() != B200BICGSTAB_RUNNING) return;
    double acc[2] = {0, 0};
    const int64_t stride = (int64_t)gridDim.x * BLOCK * 2;
    for (int64_t i = ((int64_t)blockIdx.x * BLOCK + threadIdx.x) * 2; i < n; i += stride) {
        if (i + 1 < n) {
            const double2 tt = *reinterpret_cast<const double2*>(t + i), ss = *reinterpret_cast<const double2*>(s + i);
            acc[0] += tt.x * ss.x + tt.y * ss.y;
            acc[1] += tt.x * tt.x + tt.y * tt.y;
        } else {
            acc[0] += t[i] * s[i];
            acc[1] += t[i] * t[i];
        }
    }
    block_sum_k<2>(acc, sred);
    if (threadIdx.x == 0) grid_sum_finish_k<2>(acc, ws, state + B200BICGSTAB_TS);
}

// converged at s (sqrt(s2) < threshold): x += alpha p;  r = s.   Otherwise omega = ts / tt;  x += alpha p + omega s;
// r = s - omega t.  Both: rho_new = r0 . r and r2 = r . r; the last CTA publishes omega, or the status, counter and history.
__global__ void __launch_bounds__(BLOCK) update_xr_kernel(int64_t n, double* __restrict__ x, double* __restrict__ r,
                                                          const double* __restrict__ p, const double* __restrict__ s,
                                                          const double* __restrict__ t, const double* __restrict__ r0,
                                                          double* __restrict__ state, double* __restrict__ ws) {
    __shared__ double sred[2 * (BLOCK / 32)];
    const State st(state);
    if (st.status() != B200BICGSTAB_RUNNING) return;
    const double s2 = state[B200BICGSTAB_S2], ts = state[B200BICGSTAB_TS], tt = state[B200BICGSTAB_TT];
    const double alpha = state[B200BICGSTAB_ALPHA];
    const bool conv = isfinite(s2) && below(s2, state[B200BICGSTAB_THRESHOLD]);
    double omega = 0;
    int stop = B200BICGSTAB_RUNNING;         // a breakdown: nothing is updated
    if (!isfinite(s2)) {
        stop = B200BICGSTAB_BREAKDOWN_NONFINITE;
    } else if (!conv) {
        omega = ts / tt;
        stop = !isfinite(ts) || !isfinite(tt) ? B200BICGSTAB_BREAKDOWN_NONFINITE
             : tt == 0                        ? B200BICGSTAB_BREAKDOWN_TT
             : !isfinite(omega)               ? B200BICGSTAB_BREAKDOWN_NONFINITE
             : omega == 0                     ? B200BICGSTAB_BREAKDOWN_OMEGA
                                              : B200BICGSTAB_RUNNING;
    }
    if (stop != B200BICGSTAB_RUNNING) {
        if (blockIdx.x == 0 && threadIdx.x == 0) st.status() = stop;
        return;
    }
    double acc[2] = {0, 0};
    const int64_t stride = (int64_t)gridDim.x * BLOCK * 2;
    for (int64_t i = ((int64_t)blockIdx.x * BLOCK + threadIdx.x) * 2; i < n; i += stride) {
        if (i + 1 < n) {
            const double2 pp = *reinterpret_cast<const double2*>(p + i), ss = *reinterpret_cast<const double2*>(s + i);
            const double2 q = *reinterpret_cast<const double2*>(r0 + i);
            double2 xx = *reinterpret_cast<double2*>(x + i), rr;
            if (conv) {
                xx.x += alpha * pp.x; xx.y += alpha * pp.y;
                rr = ss;
            } else {
                const double2 tv = *reinterpret_cast<const double2*>(t + i);
                xx.x = (xx.x + alpha * pp.x) + omega * ss.x; xx.y = (xx.y + alpha * pp.y) + omega * ss.y;
                rr.x = ss.x - omega * tv.x; rr.y = ss.y - omega * tv.y;
            }
            *reinterpret_cast<double2*>(x + i) = xx;
            *reinterpret_cast<double2*>(r + i) = rr;
            acc[0] += q.x * rr.x + q.y * rr.y;
            acc[1] += rr.x * rr.x + rr.y * rr.y;
        } else {
            double rn;
            if (conv) {
                x[i] += alpha * p[i];
                rn = s[i];
            } else {
                x[i] = (x[i] + alpha * p[i]) + omega * s[i];
                rn = s[i] - omega * t[i];
            }
            r[i] = rn;
            acc[0] += r0[i] * rn;
            acc[1] += rn * rn;
        }
    }
    block_sum_k<2>(acc, sred);
    if (threadIdx.x == 0 && grid_sum_finish_k<2>(acc, ws, state + B200BICGSTAB_RHO_NEW)) {
        if (conv) {
            st.finish_iteration(s2);
            st.status() = B200BICGSTAB_CONVERGED_S;
        } else {
            state[B200BICGSTAB_OMEGA] = omega;
        }
    }
}

// converged at r (sqrt(r2) < threshold), rho_new = 0 or a non-finite scalar: p is left as it is.  Otherwise
// beta = (rho_new / rho) (alpha / omega);  p = r + beta (p - omega v).  Both count the iteration.
__global__ void __launch_bounds__(BLOCK) update_p_kernel(int64_t n, double* __restrict__ p, const double* __restrict__ r,
                                                         const double* __restrict__ v, double* __restrict__ state) {
    const State st(state);
    if (st.status() != B200BICGSTAB_RUNNING) return;
    const double rho_new = state[B200BICGSTAB_RHO_NEW], r2 = state[B200BICGSTAB_R2], omega = state[B200BICGSTAB_OMEGA];
    const double beta = (rho_new / state[B200BICGSTAB_RHO]) * (state[B200BICGSTAB_ALPHA] / omega);
    const int next = !isfinite(r2) || !isfinite(rho_new)          ? B200BICGSTAB_BREAKDOWN_NONFINITE
                   : below(r2, state[B200BICGSTAB_THRESHOLD])     ? B200BICGSTAB_CONVERGED_R
                   : rho_new == 0                                 ? B200BICGSTAB_BREAKDOWN_RHO
                   : !isfinite(beta)                              ? B200BICGSTAB_BREAKDOWN_NONFINITE
                                                                  : B200BICGSTAB_RUNNING;
    if (blockIdx.x == 0 && threadIdx.x == 0) {
        st.finish_iteration(r2);
        if (next != B200BICGSTAB_RUNNING) st.status() = next;
    }
    if (next != B200BICGSTAB_RUNNING) return;
    const int64_t stride = (int64_t)gridDim.x * BLOCK * 2;
    for (int64_t i = ((int64_t)blockIdx.x * BLOCK + threadIdx.x) * 2; i < n; i += stride) {
        if (i + 1 < n) {
            const double2 rr = *reinterpret_cast<const double2*>(r + i), vv = *reinterpret_cast<const double2*>(v + i);
            double2 pp = *reinterpret_cast<double2*>(p + i);
            pp.x = rr.x + beta * (pp.x - omega * vv.x); pp.y = rr.y + beta * (pp.y - omega * vv.y);
            *reinterpret_cast<double2*>(p + i) = pp;
        } else {
            p[i] = r[i] + beta * (p[i] - omega * v[i]);
        }
    }
}

}  // namespace b200bicgstab

using namespace b200bicgstab;

extern "C" {

size_t b200bicgstab_workspace_bytes(void) { return (size_t)(WS_STRIDE + MAX_CTAS) * sizeof(double); }

size_t b200bicgstab_state_layout(int64_t history_len, int32_t* status_byte, int32_t* iter_byte, int32_t* history_byte) {
    if (status_byte) *status_byte = STATUS_BYTE;
    if (iter_byte) *iter_byte = ITER_BYTE;
    if (history_byte) *history_byte = HEADER_BYTES;
    if (history_len < 0 || history_len > INT32_MAX) return 0;
    return HEADER_BYTES + (size_t)history_len * sizeof(double);
}

int b200bicgstab_init(void* stream, int64_t n, const double* r0, double* r, double* p, void* state, int64_t history_len, double tol) {
    if (n < 0 || !state || (n > 0 && (!r0 || !r || !p)) || !aligned16(r0) || !aligned16(r) || !aligned16(p) || !aligned16(state)) return -1;
    if (history_len < 0 || history_len > INT32_MAX || isnan(tol)) return -1;
    init_kernel<<<grid_for(n), BLOCK, 0, (cudaStream_t)stream>>>(n, r0, r, p, (double*)state, (int32_t)history_len, tol);
    return (int)cudaGetLastError();
}

int b200bicgstab_update_s(void* stream, int64_t n, const double* r, const double* v, double* s, void* state, void* workspace) {
    if (n < 0 || !state || !workspace || (n > 0 && (!r || !v || !s)) || !aligned16(r) || !aligned16(v) || !aligned16(s) || !aligned16(state)) return -1;
    update_s_kernel<<<grid_for(n), BLOCK, 0, (cudaStream_t)stream>>>(n, r, v, s, (double*)state, (double*)workspace);
    return (int)cudaGetLastError();
}

int b200bicgstab_dot2(void* stream, int64_t n, const double* t, const double* s, void* state, void* workspace) {
    if (n < 0 || !state || !workspace || (n > 0 && (!t || !s)) || !aligned16(t) || !aligned16(s) || !aligned16(state)) return -1;
    dot2_kernel<<<grid_for(n), BLOCK, 0, (cudaStream_t)stream>>>(n, t, s, (double*)state, (double*)workspace);
    return (int)cudaGetLastError();
}

int b200bicgstab_update_xr(void* stream, int64_t n, double* x, double* r, const double* p, const double* s, const double* t,
                           const double* r0, void* state, void* workspace) {
    if (n < 0 || !state || !workspace || (n > 0 && (!x || !r || !p || !s || !t || !r0))) return -1;
    if (!aligned16(x) || !aligned16(r) || !aligned16(p) || !aligned16(s) || !aligned16(t) || !aligned16(r0) || !aligned16(state)) return -1;
    update_xr_kernel<<<grid_for(n), BLOCK, 0, (cudaStream_t)stream>>>(n, x, r, p, s, t, r0, (double*)state, (double*)workspace);
    return (int)cudaGetLastError();
}

int b200bicgstab_update_p(void* stream, int64_t n, double* p, const double* r, const double* v, void* state) {
    if (n < 0 || !state || (n > 0 && (!p || !r || !v)) || !aligned16(p) || !aligned16(r) || !aligned16(v) || !aligned16(state)) return -1;
    update_p_kernel<<<grid_for(n), BLOCK, 0, (cudaStream_t)stream>>>(n, p, r, v, (double*)state);
    return (int)cudaGetLastError();
}

}  // extern "C"
