// batched_banded.cuh -- the kernels of batched_banded.cu: many small banded systems A_j x_j = b_j solved at once, one thread per
// system, in the interleaved layout of cusparse<t>gpsvInterleavedBatch / gtsvInterleavedBatch (element i of system j at
// i * batch + j, so a warp's loads and stores are coalesced).  The launches are in batched_banded.cu; this header is also compiled
// for the host by tests/host_emulation/emulate_banded.cpp, so it uses no device-only intrinsic.  DESIGN.md 3.25.
//
// One sweep serves every method.  A system with P sub-diagonals (P = 2: gpsv's ds, dl; P = 1: gtsv's dl) keeps a window of P + 1
// rows in registers, each row 2P + 1 columns wide starting at the column k being eliminated:
//   step k   eliminate column k of rows k + 1 .. k + P against row k (Givens rotations, or pivoted / plain Gaussian elimination);
//            row k is then row k of the triangular factor U: its diagonal u and up to W entries to the right.  Write
//            U[k][1..W] / u to the workspace and b'[k] / u over x[k] (x[k] has been read: the right-hand side of row k);
//   shift    the window moves one column right and one row down: row k + 1 + P is read from the coefficient arrays.
// Back substitution walks k = m - 1 .. 0: x[k] -= sum_j (U[k][j] / u) x[k + j], the last W solutions kept in registers.
//   gpsv (algo 0), gtsv algo 2   Givens QR: W = 2P (R's upper bandwidth 2P: 4 for gpsv, 2 for gtsv).  Complex rotations have a
//                                real c and a complex s: [c  s; -conj(s)  c].
//   gtsv algo 1                  LU with partial pivoting between rows k and k + 1: W = 2 (one superdiagonal of fill).
//   gtsv algo 0                  Thomas, no pivoting: W = 1.  Unstable by design, as the closed library's algo 0 is.
// The coefficient arrays are only read, and their out-of-band slots (ds[0..1], dl[0], du[m-1], dw[m-2..m-1]) never: rows and columns
// outside the matrix are zeros, so a rotation or an elimination against them is the identity.  No atomics, no cross-thread
// communication: each system's result is a pure function of its inputs.  Workspace: W * m * batch values, U[k][q] of system j at
// (k * W + q - 1) * batch + j.
#pragma once
#include <cmath>
#include <cstdint>

namespace b200 {

// The value types: float, double, and cplx<float> / cplx<double> with cuComplex / cuDoubleComplex's layout.
template <typename R>
struct alignas(2 * sizeof(R)) cplx {
    R re, im;
};

template <typename T> struct real_of { using type = T; };
template <typename R> struct real_of<cplx<R>> { using type = R; };

__device__ __forceinline__ float bb_hypot(float a, float b) { return hypotf(a, b); }
__device__ __forceinline__ double bb_hypot(double a, double b) { return hypot(a, b); }

template <typename R> __device__ __forceinline__ R bb_abs(R a) { return a < R(0) ? -a : a; }
template <typename R> __device__ __forceinline__ R bb_abs(cplx<R> a) { return bb_hypot(a.re, a.im); }
template <typename R> __device__ __forceinline__ R bb_abs1(R a) { return bb_abs(a); }
template <typename R> __device__ __forceinline__ R bb_abs1(cplx<R> a) { return bb_abs(a.re) + bb_abs(a.im); }   // LAPACK's cabs1
template <typename R> __device__ __forceinline__ bool bb_zero(R a) { return a == R(0); }
template <typename R> __device__ __forceinline__ bool bb_zero(cplx<R> a) { return a.re == R(0) && a.im == R(0); }
template <typename R> __device__ __forceinline__ R bb_conj(R a) { return a; }
template <typename R> __device__ __forceinline__ cplx<R> bb_conj(cplx<R> a) { return {a.re, -a.im}; }
template <typename R> __device__ __forceinline__ R bb_mul(R a, R b) { return a * b; }
template <typename R> __device__ __forceinline__ cplx<R> bb_mul(cplx<R> a, cplx<R> b) {
    return {a.re * b.re - a.im * b.im, a.re * b.im + a.im * b.re};
}
template <typename R> __device__ __forceinline__ R bb_scale(R c, R a) { return c * a; }
template <typename R> __device__ __forceinline__ cplx<R> bb_scale(R c, cplx<R> a) { return {c * a.re, c * a.im}; }
template <typename R> __device__ __forceinline__ R bb_add(R a, R b) { return a + b; }
template <typename R> __device__ __forceinline__ cplx<R> bb_add(cplx<R> a, cplx<R> b) { return {a.re + b.re, a.im + b.im}; }
template <typename R> __device__ __forceinline__ R bb_sub(R a, R b) { return a - b; }
template <typename R> __device__ __forceinline__ cplx<R> bb_sub(cplx<R> a, cplx<R> b) { return {a.re - b.re, a.im - b.im}; }
template <typename V> __device__ __forceinline__ V bb_one() { V v{}; reinterpret_cast<typename real_of<V>::type*>(&v)[0] = 1; return v; }
// a / d for a real d, part by part: never through 1 / d, which overflows for a subnormal d
template <typename R> __device__ __forceinline__ R bb_rdiv(R a, R d) { return a / d; }
template <typename R> __device__ __forceinline__ cplx<R> bb_rdiv(cplx<R> a, R d) { return {a.re / d, a.im / d}; }
// top / |top| for |top| = at > 0: the sign of a real top, top's parts over at for a complex one
template <typename R> __device__ __forceinline__ R bb_phase(R top, R) { return top < R(0) ? R(-1) : R(1); }
template <typename R> __device__ __forceinline__ cplx<R> bb_phase(cplx<R> top, R at) { return bb_rdiv(top, at); }
// a / b; the complex one by Smith's method, so that neither |b|^2 nor 1 / b is formed (no overflow or underflow on the way)
template <typename R> __device__ __forceinline__ R bb_div(R a, R b) { return a / b; }
template <typename R> __device__ __forceinline__ cplx<R> bb_div(cplx<R> a, cplx<R> b) {
    if (bb_abs(b.re) >= bb_abs(b.im)) {
        const R r = b.im / b.re, d = b.re + b.im * r;
        return {(a.re + a.im * r) / d, (a.im - a.re * r) / d};
    }
    const R r = b.re / b.im, d = b.re * r + b.im;
    return {(a.re * r + a.im) / d, (a.im * r - a.re) / d};
}

enum BandMethod { BAND_GIVENS = 0, BAND_PIVOT_LU = 1, BAND_THOMAS = 2 };

// Entries of U kept right of the diagonal: Givens and pivoted LU fill up to 2P, Thomas none past the band.
template <int P, int METHOD> struct band_width { static constexpr int W = METHOD == BAND_THOMAS ? P : 2 * P; };

template <typename V>
struct BandArgs {
    const V* diag[5];   // sub-diagonals first: P = 2 (ds, dl, d, du, dw), P = 1 (dl, d, du) in diag[0..2]
    V*       x;         // the right-hand sides in, the solutions out
    V*       work;      // W * m * batch values
    int64_t  m, batch;
};

// Row i of system j as window columns i - P .. i + P; rows outside [0, m) and out-of-band slots are zero and are not read.
template <typename V, int P>
__device__ __forceinline__ void band_load_row(const BandArgs<V>& a, int64_t i, int64_t j, V* row, V* rhs) {
    #pragma unroll
    for (int o = 0; o <= 2 * P; o++) {
        const int64_t c = i - P + o;
        row[o] = (i < a.m && c >= 0 && c < a.m) ? a.diag[o][i * a.batch + j] : V{};
    }
    *rhs = i < a.m ? a.x[i * a.batch + j] : V{};
}

// Zero r[q][0] against r[0][0]: a rotation, a pivot-and-eliminate, or a plain elimination, on both rows and their right-hand sides.
template <typename V, int P, int METHOD>
__device__ __forceinline__ void band_eliminate(V (&r)[P + 1][2 * P + 1], V (&b)[P + 1], int q) {
    using R = typename real_of<V>::type;
    const V top = r[0][0], bot = r[q][0];
    if (bb_zero(bot)) return;                       // nothing to eliminate: the identity, bit for bit
    if (METHOD == BAND_GIVENS) {
        // [c  s; -conj(s)  c] [top; bot] = [rho; 0] with c = |top| / n, s = (top / |top|) conj(bot) / n, n = |(top, bot)|
        const R at = bb_abs(top), n = bb_hypot(at, bb_abs(bot));
        const R c = at / n;
        // divisions, not reciprocals: 1 / |top| overflows for a subnormal top; both quotients have modulus at most 1
        const V ph = at == R(0) ? bb_one<V>() : bb_phase(top, at);        // top / |top|, or 1 when top = 0
        const V s = bb_mul(ph, bb_rdiv(bb_conj(bot), n));
        const V ms = bb_sub(V{}, bb_conj(s));
        #pragma unroll
        for (int c2 = 0; c2 <= 2 * P; c2++) {
            const V p = r[0][c2], t = r[q][c2];
            r[0][c2] = bb_add(bb_scale(c, p), bb_mul(s, t));
            r[q][c2] = bb_add(bb_mul(ms, p), bb_scale(c, t));
        }
        r[q][0] = V{};
        const V p = b[0], t = b[q];
        b[0] = bb_add(bb_scale(c, p), bb_mul(s, t));
        b[q] = bb_add(bb_mul(ms, p), bb_scale(c, t));
    } else {
        if (METHOD == BAND_PIVOT_LU && bb_abs1(bot) > bb_abs1(top)) {
            #pragma unroll
            for (int c2 = 0; c2 <= 2 * P; c2++) { const V t = r[0][c2]; r[0][c2] = r[q][c2]; r[q][c2] = t; }
            const V t = b[0]; b[0] = b[q]; b[q] = t;
        }
        const V l = bb_div(r[q][0], r[0][0]);
        #pragma unroll
        for (int c2 = 1; c2 <= 2 * P; c2++) r[q][c2] = bb_sub(r[q][c2], bb_mul(l, r[0][c2]));
        r[q][0] = V{};
        b[q] = bb_sub(b[q], bb_mul(l, b[0]));
    }
}

template <typename V, int P, int METHOD>
__device__ __forceinline__ void band_solve_system(const BandArgs<V>& a, int64_t j) {
    constexpr int W = band_width<P, METHOD>::W;
    V r[P + 1][2 * P + 1], b[P + 1];
    #pragma unroll
    for (int q = 0; q <= P; q++) {
        #pragma unroll
        for (int c = 0; c <= 2 * P; c++) r[q][c] = V{};
        b[q] = V{};
    }
    // shift: the window moves one column right and one row down, row i enters at the bottom
    auto shift_in = [&](int64_t i) {
        #pragma unroll
        for (int q = 0; q < P; q++) {
            #pragma unroll
            for (int c = 0; c < 2 * P; c++) r[q][c] = r[q + 1][c + 1];
            r[q][2 * P] = V{};
            b[q] = b[q + 1];
        }
        band_load_row<V, P>(a, i, j, r[P], &b[P]);
    };
    #pragma unroll
    for (int i = 0; i <= P; i++) shift_in(i);       // from the all-zero window left of column 0: rows 0 .. P at column 0
    for (int64_t k = 0; k < a.m; k++) {
        #pragma unroll
        for (int q = 1; q <= P; q++) band_eliminate<V, P, METHOD>(r, b, q);
        #pragma unroll
        for (int q = 1; q <= W; q++) a.work[(k * W + q - 1) * a.batch + j] = bb_div(r[0][q], r[0][0]);
        a.x[k * a.batch + j] = bb_div(b[0], r[0][0]);
        shift_in(k + 1 + P);
    }
    V xs[W];                                        // x[k + 1 .. k + W]; zero past the matrix
    #pragma unroll
    for (int q = 0; q < W; q++) xs[q] = V{};
    for (int64_t k = a.m - 1; k >= 0; k--) {
        V v = a.x[k * a.batch + j];
        #pragma unroll
        for (int q = 1; q <= W; q++)
            if (k + q < a.m) v = bb_sub(v, bb_mul(a.work[(k * W + q - 1) * a.batch + j], xs[q - 1]));
        a.x[k * a.batch + j] = v;
        #pragma unroll
        for (int q = W - 1; q > 0; q--) xs[q] = xs[q - 1];
        xs[0] = v;
    }
}

constexpr int BAND_BLOCK = 128;

template <typename V, int P, int METHOD>
__global__ void __launch_bounds__(BAND_BLOCK) banded_interleaved_kernel(BandArgs<V> a) {
    const int64_t j = (int64_t)blockIdx.x * BAND_BLOCK + threadIdx.x;
    if (j < a.batch) band_solve_system<V, P, METHOD>(a, j);
}

}  // namespace b200
