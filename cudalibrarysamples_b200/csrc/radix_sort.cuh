// radix_sort.cuh -- the stable LSD radix sort of spmm_csr_t.cu (DESIGN.md 3.22), shared with the conversions of convert.cu (3.23).
//
// One host-side driver over the transposed plan's three kernels per pass (digit histogram per RT_TILE-entry tile, per-digit scan,
// stable scatter), plus the passes built on a sorted key array: column pointers, the row of each entry, and a bit-exact gather of
// values by a permutation.  Everything runs on the caller's stream in the caller's memory: no allocation, no host synchronisation.
#pragma once

#include <cstddef>
#include <cstdint>

#include <cuda_runtime.h>

namespace b200 {

constexpr int RT_THREADS = 256;                    // threads of every sort kernel
constexpr int RT_ITEMS = 8;                        // entries per thread per pass: one round of RT_THREADS entries each
constexpr int RT_TILE = RT_THREADS * RT_ITEMS;     // entries per tile
constexpr int RT_BITS = 8, RT_BINS = 1 << RT_BITS;

// The sort's scratch for n entries: two key buffers, two index buffers (each 256-byte aligned, n ints), the tile histograms and the
// digit totals, in this order from one 256-byte aligned base.
struct RtScratch {
    int* k[2];
    int* v[2];
    int* hist;
    int* tot;
};
size_t rt_scratch_bytes(int64_t n);
RtScratch rt_scratch(char* base, int64_t n);

// Passes for keys in [0, nkeys): as many 8-bit digits as nkeys - 1 needs, at least one.
int rt_passes(int64_t nkeys);

// Stable sort of the entries 0 .. n-1 by key, where entry i has key keys[kidx ? kidx[i] : i] - sub and carries the index
// vals ? vals[i] : i.  Keys outside [0, nkeys) are sorted by their low rt_passes(nkeys) digits only, and nothing is written outside
// the outputs.  The sorted keys go to s.k[(passes - 1) & 1]; the carried indices to vals_out, or to s.v[(passes - 1) & 1] when
// vals_out is NULL.  vals_out must not be the index buffer the last pass reads (s.v[passes & 1] when passes > 1, else vals).  On
// return *sorted_keys / *sorted_vals (either may be NULL) point at the results.  n > 0.
void rt_sort(cudaStream_t st, const int* keys, int sub, const int* kidx, const int* vals, int n, int64_t nkeys, const RtScratch& s,
             int* vals_out, const int** sorted_keys, const int** sorted_vals);

// out[c] = base + (the first k with keys[k] - sub >= c), for c in [0, nkeys]: column pointers from sorted keys.  Writes stay in
// out[0 .. nkeys] whatever the keys hold.
void rt_offsets(cudaStream_t st, const int* keys, int sub, int n, int64_t nkeys, int base, int* out);

// out[k] = out_base + (the row r with off[r] - off_base <= (perm ? perm[k] : k), the last such), a binary search in rows >= 1
// offsets.  Writes stay in out[0 .. n).
void rt_rows(cudaStream_t st, const int* off, int off_base, int64_t rows, const int* perm, int n, int out_base, int* out);

// dst[k] = src[perm[k]] for k < n, bit for bit, elements of `width` bytes (1, 2, 4, 8 or 16).  False on another width.
bool rt_gather(cudaStream_t st, int width, const void* src, const int* perm, int n, void* dst);

}  // namespace b200
