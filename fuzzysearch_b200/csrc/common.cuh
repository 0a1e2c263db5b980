// common.cuh -- shared declarations for the libfuzzb200 kernels (sm_90a).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "fuzzb200.h"

namespace fzb {

constexpr int kMaxPattern = FZB_MAX_PATTERN;
constexpr int kGranuleShift = 6;  // verify granule = 64 anchor positions
constexpr int kGranule = 1 << kGranuleShift;

// One raw match as emitted by the verify kernels.
struct RawRec {
    int64_t start;
    int64_t end;
    int64_t idx;     // anchor: n-gram hit index (n-gram routes) / start (others)
    int32_t dist;
    int32_t ngram;   // n-gram ordinal (n-gram routes); multiplicity (LP routes)
};

// Everything a scan/verify kernel needs, passed by value (kernel parameter space).
struct ScanParams {
    const uint8_t *H;   // device buffer; H[0] is global position buf_lo
    int64_t buf_lo;     // global position of H[0]
    int64_t buf_len;    // valid bytes in the buffer
    int64_t N;          // global sequence length (window clipping happens at 0 and N only)
    int64_t own_lo;     // anchors owned by this shard: [own_lo, own_hi)
    int64_t own_hi;
    uint32_t *bitmap;   // dirty-granule bitmap, bit g <-> buffer offsets [64g, 64g+64)
    uint32_t *glist;    // work list of marked granules, appended by whoever flips a bitmap bit 0 -> 1
    uint32_t glist_cap;
    uint32_t *counters; // CNT_* slots
    uint64_t *hits;     // dense filter, hit-list mode: confirmed n-gram hits (idx << 8 | n-gram ordinal)
    uint32_t hits_cap;  // 0 = mark granules instead
    int32_t m, k, L, n_ngrams;
    int32_t q;          // bytes per hashed sample (4 sampled filter; min(L,4) dense filter)
    int32_t max_subs, max_ins, max_dels;  // generic route only
    uint8_t P[256];     // the pattern
};

// counters[] slots (device, uint32 each unless noted)
enum { CNT_OUT = 0, CNT_CAND = 1, CNT_OVERFLOW = 2, CNT_GRAN = 3, CNT_WORK = 4, /* 5,6: post_kernels.cuh */
       CNT_HITS = 7, CNT_HITWORK = 8, /* 9: post_kernels.cuh */ CNT_KEYS = 14, CNT_COUNT = 16 };

// A record set (fzb_haystack_set_records, DESIGN.md section 5.10): record r of a whole-sequence buffer is
// [off[r], off[r+1] - 1), followed by one separator position off[r+1] - 1.  first[g] is the record that holds position
// 64 g.  Only the exact stages read it, through rec_bounds; kernels take it as a trailing argument and ignore it in
// their REC == false instantiations.
struct RecSet {
    const uint64_t *off;
    const uint32_t *first;
};

// [lo, hi) of the record holding buffer position x (x < N); false if x is that record's separator (x == hi).  A
// 64-position granule holds at most 64 record starts, so the walk from first[] takes at most 64 steps.
__device__ __forceinline__ bool rec_bounds(const RecSet &rs, int64_t x, int64_t &lo, int64_t &hi) {
    uint32_t r = rs.first[x >> kGranuleShift];
    while ((int64_t)rs.off[r + 1] <= x) r++;
    lo = (int64_t)rs.off[r];
    hi = (int64_t)rs.off[r + 1] - 1;
    return x < hi;
}

// first[g] for every granule g < ngran: the largest r with off[r] <= 64 g (binary search over the count + 1 offsets)
__global__ void k_rec_first(const uint64_t *off, uint64_t count, uint32_t *first, uint64_t ngran) {
    const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
    for (uint64_t g = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; g < ngran; g += stride) {
        const uint64_t x = g << kGranuleShift;
        uint64_t lo = 0, hi = count;  // off[lo] <= x < off[hi]
        while (hi - lo > 1) {
            const uint64_t mid = (lo + hi) / 2;
            if (off[mid] <= x) lo = mid; else hi = mid;
        }
        first[g] = (uint32_t)lo;
    }
}

__host__ __device__ __forceinline__ uint64_t splitmix64(uint64_t x) {
    x += 0x9E3779B97F4A7C15ull;
    x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ull;
    x = (x ^ (x >> 27)) * 0x94D049BB133111EBull;
    return x ^ (x >> 31);
}

// Synthetic corpus: bytes 4q..4q+3 come from one 64-bit hash of (seed, q): 16 bits per byte.
__host__ __device__ __forceinline__ uint32_t synth_word(uint64_t seed, uint64_t q,
                                                         const uint8_t *alphabet, uint32_t alen) {
    uint64_t x = splitmix64(seed ^ (q * 0xD1342543DE82EF95ull));
    uint32_t w = 0;
#pragma unroll
    for (int b = 0; b < 4; b++) {
        uint32_t r = (uint32_t)(x >> (16 * b)) & 0xFFFFu;
        w |= (uint32_t)alphabet[(r * alen) >> 16] << (8 * b);
    }
    return w;
}

}  // namespace fzb
