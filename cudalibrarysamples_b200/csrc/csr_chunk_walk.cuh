// csr_chunk_walk.cuh -- the chunked CSR SpMV walk, y = alpha * A * x + beta * y, shared by spmv_csr16.cu (fp16 / bf16 values, fp32
// sums) and the opA = N path of spmv_csr_z.cu (double complex).  Everything here has internal linkage or is inlined into the
// kernels of those files, which keep their own names and launch bounds.
//
// Plan-free and balanced by entries: no preprocess, so the cg / bicgstab call pattern (bufferSize, then SpMV, never preprocess) gets
// the same kernel.  The entry range is cut into chunks of E = P::CHUNK entries at fixed positions: chunk c is [c * E, (c + 1) * E).
// One warp takes one chunk:
//   * it finds the chunk's first row with one binary search over the offsets;
//   * it streams the chunk's columns and values, gathers x and parks the products in shared memory (P::products);
//   * a lane sums each run of R = P::RUN products (the chunk's entries [R q, R q + R)) in order, from 0;
//   * one lane per row then adds the row's piece -- the part of the row inside the chunk -- run by run in ascending order, from 0:
//     a run the piece covers whole contributes its run sum, a run it covers in part contributes 0 + its products in order.
// So the piece sum S(r, c) depends only on the piece's products and its start and end inside the chunk: not on other rows, the grid
// or the SM count.  The row total is acc_r = ((0 + S(r, c0)) + S(r, c0 + 1)) + ..., the pieces in ascending chunk order, and P::store
// writes y_r = alpha * acc_r + beta * y_r (beta == 0 never reads y; an empty row gets beta * y).  The "0 +" is explicit everywhere:
// it turns -0 into +0, and both walks below must agree on it.
//
// Split walk (a workspace of csr_walk_carry_bytes): a row that starts and ends in one chunk is written by that chunk's warp.  Each
// chunk has two carry slots: in[c] for the piece of the row that enters it from an earlier chunk (at most one), out[c] for the piece
// of the row that starts in c and leaves it (at most one).  The fix-up kernel owns each such row at its starting chunk: it adds
// out[c], then in[c + 1], in[c + 2], ... and writes y once.  Every slot is written once and read once.
// Unsplit walk (no usable workspace): the warp of a row's starting chunk computes the row's later pieces itself with the same piece
// code and adds them in the same order.  This serialises hub rows, but both walks give identical bits.  No atomics, no allocation,
// no host synchronisation: repeated calls and graph replays give identical bits.
//
// Nothing past nnz is loaded; x is read only at stored columns.
//
// The policy P of an element type provides:
//   Args                     the kernel arguments: off, rows, base, nchunks and carry (Acc*: in[c] = carry[2c],
//                            out[c] = carry[2c + 1]; nullptr = unsplit), plus what products and store read
//   Acc                      the accumulator type
//   WARPS, CHUNK, RUN        warps (= chunks) per CTA, E and R
//   zero(), add(u, v)        0 and the correctly rounded sum
//   shfl(v, src)             v of lane src, to the whole warp
//   slot(p)                  where chunk position p lives in a warp's product array
//   products(a, c, lane, prod, runs)   chunk c's products into prod (0 past nnz), then the run sums 0 + p0 + ... into runs
//   store(a, r, acc, alpha, beta)      y_r = alpha * acc + beta * y_r
#pragma once
#include "spmv_common.cuh"

namespace b200 {

constexpr int CSR_WALK_FIXUP_THREADS = 256;           // one thread per chunk

template <class Args>
__device__ __forceinline__ int csr_off(const Args& a, int r) { return __ldg(a.off + r) - a.base; }

// the first row starting at or after entry e (off[rows] = nnz >= e)
template <class Args>
__device__ __forceinline__ int csr_first_row(const Args& a, int e) {
    int lo = 0, hi = a.rows;
    while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (csr_off(a, mid) < e) lo = mid + 1; else hi = mid;
    }
    return lo;
}

// S of the piece [s, e) (chunk coordinates): 0 + its runs' sums in ascending order; a run covered in part adds 0 + its products in order
template <class P>
__device__ __forceinline__ typename P::Acc csr_walk_piece(const typename P::Acc* prod, const typename P::Acc* runs, int s, int e) {
    typename P::Acc acc = P::zero();
    for (int p = s; p < e;) {
        const int q = min(e, (p / P::RUN + 1) * P::RUN);
        typename P::Acc u;
        if (q - p == P::RUN) {
            u = runs[p / P::RUN];
        } else {
            u = P::zero();
            for (int i = p; i < q; i++) u = P::add(u, prod[P::slot(i)]);
        }
        acc = P::add(acc, u);
        p = q;
    }
    return acc;
}

// The chunk kernel's body.  One warp per chunk.  Rows handled: the one entering the chunk from an earlier chunk (its piece goes to
// in[c]) and the rows that start in the chunk (the last chunk also takes the empty rows at nnz); of those, the one leaving the chunk
// goes to out[c].  sprod / sruns: the CTA's shared product and run-sum arrays, one row per warp.  a and sc come by value, as the
// kernel's own parameters do: by reference, the double-complex kernel compiles to different SASS.
template <class P>
__device__ __forceinline__ void csr_walk_chunk(const typename P::Args a, const Scalars<typename P::Acc> sc,
                                               typename P::Acc (*sprod)[P::CHUNK], typename P::Acc (*sruns)[P::CHUNK / P::RUN]) {
    using Acc = typename P::Acc;
    const int lane = (int)threadIdx.x & 31, warp = (int)threadIdx.x >> 5;
    const int c = (int)blockIdx.x * P::WARPS + warp;
    if (c >= a.nchunks) return;
    Acc* prod = sprod[warp];
    Acc* runs = sruns[warp];
    const int cs = c * P::CHUNK, ce = cs + P::CHUNK;
    const bool last = c == a.nchunks - 1;
    const int lo = csr_first_row(a, cs);
    P::products(a, c, lane, prod, runs);
    const Acc alpha = sc.a(), beta = sc.b();
    const int r0 = lo > 0 && csr_off(a, lo) > cs ? lo - 1 : lo;   // the row entering the chunk, if one does
    int leave_row = -1;
    Acc leave_s = P::zero();
    for (int rb = r0;; rb += 32) {                      // warp-uniform: 32 rows at a time while every lane has one of ours
        const int r = rb + lane;
        int rs = 0, re = 0;
        bool live = r < a.rows;
        if (live) {
            rs = csr_off(a, r);
            live = last || rs < ce;
        }
        if (live) {
            re = csr_off(a, r + 1);
            const Acc s = csr_walk_piece<P>(prod, runs, max(rs, cs) - cs, min(re, ce) - cs);
            if (rs < cs) {                              // the entering row: the fix-up's (split) or its owner's (unsplit)
                if (a.carry) a.carry[2 * c] = s;
            } else if (re > ce) {                       // the leaving row
                if (a.carry) a.carry[2 * c + 1] = s;
                leave_row = r; leave_s = s;
            } else {
                P::store(a, r, P::add(P::zero(), s), alpha, beta);
            }
        }
        if (!__all_sync(0xffffffffu, live)) break;
    }
    if (a.carry) return;
    // unsplit: this warp adds the leaving row's later pieces itself, in chunk order, with the same piece code
    const unsigned who = __ballot_sync(0xffffffffu, leave_row >= 0);
    if (!who) return;
    const int src = __ffs(who) - 1;
    const int r = __shfl_sync(0xffffffffu, leave_row, src);
    Acc acc = P::add(P::zero(), P::shfl(leave_s, src));
    const int re = csr_off(a, r + 1);
    for (int c2 = c + 1; c2 * P::CHUNK < re; c2++) {
        __syncwarp();                                   // every lane is done with the previous chunk's products
        P::products(a, c2, lane, prod, runs);
        if (lane == 0) acc = P::add(acc, csr_walk_piece<P>(prod, runs, 0, min(re - c2 * P::CHUNK, P::CHUNK)));
    }
    if (lane == 0) P::store(a, r, acc, alpha, beta);
}

// The fix-up kernel's body (split walk, part 2): the row that starts in chunk c and leaves it (at most one) gets
// 0 + out[c] + in[c + 1] + in[c + 2] + ..., in ascending chunk order, written once.  One thread per chunk; the last chunk has no
// such row.
template <class P>
__device__ __forceinline__ void csr_walk_fixup(const typename P::Args a, const Scalars<typename P::Acc> sc) {
    const int c = (int)blockIdx.x * CSR_WALK_FIXUP_THREADS + (int)threadIdx.x;
    if (c >= a.nchunks - 1) return;
    const int cs = c * P::CHUNK, ce = cs + P::CHUNK;
    const int r = csr_row_of(a.off, a.rows, a.base, ce - 1);   // the row holding the chunk's last entry (< nnz)
    const int rs = csr_off(a, r), re = csr_off(a, r + 1);
    if (rs < cs || re <= ce) return;                    // it starts before the chunk, or ends in it
    typename P::Acc acc = P::add(P::zero(), a.carry[2 * c + 1]);
    for (int c2 = c + 1; c2 * P::CHUNK < re; c2++) acc = P::add(acc, a.carry[2 * c2]);
    P::store(a, r, acc, sc.a(), sc.b());
}

// ------------------------------------------------------------------------------------------------ host side
template <int E>
static int64_t csr_walk_nchunks(int64_t nnz) { return nnz > 0 ? (nnz + E - 1) / E : 1; }

// the split walk's workspace: two carry slots of type Acc per chunk of E entries
template <int E, typename Acc>
static size_t csr_walk_carry_bytes(int64_t rows, int64_t nnz) {
    if (rows <= 0 || nnz <= 0) return 0;
    return 2 * (size_t)csr_walk_nchunks<E>(nnz) * sizeof(Acc);
}

// The carry slots in the caller's workspace, or nullptr for the unsplit walk: a NULL, misaligned or smaller buffer gets it, with the
// same bits.  One chunk: no row leaves it.
template <int E, typename Acc>
static Acc* csr_walk_carry(int64_t rows, int64_t nnz, void* workspace, size_t workspace_bytes) {
    const bool split = csr_walk_nchunks<E>(nnz) > 1 &&
                       workspace_usable(workspace, workspace_bytes, csr_walk_carry_bytes<E, Acc>(rows, nnz));
    return split ? (Acc*)workspace : nullptr;
}

// the chunk kernel over every chunk, then the fix-up when the walk is split
template <int WARPS, class Args, class S>
static int csr_walk_launch(cudaStream_t st, void (*chunk)(Args, S), void (*fixup)(Args, S), const Args& a, const S& sc) {
    chunk<<<(unsigned)((a.nchunks + WARPS - 1) / WARPS), 32 * WARPS, 0, st>>>(a, sc);
    constexpr int FT = CSR_WALK_FIXUP_THREADS;
    if (a.carry) fixup<<<(unsigned)((a.nchunks - 1 + FT - 1) / FT), FT, 0, st>>>(a, sc);
    return (int)cudaGetLastError();
}

}  // namespace b200
