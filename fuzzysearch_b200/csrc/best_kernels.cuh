// best_kernels.cuh -- fzb_best_per_record (DESIGN.md section 5.13): the raw records of a pass over a record set,
// reduced on the device to two words per record of the set.
//
// best[r]: the smallest key  dist (8 bits) | pattern (16) | kBestMaxLen - length (9) | start - record start (31)  of
// any raw match in record r, most significant field first: the nearest match, of the pattern with the smallest
// ordinal, the longest, the leftmost.  top2[r]: 0xFFFF | first (24 bits) | second (24 bits), the two smallest pairs
// dist (8) | pattern (16) whose patterns differ.  Nothing yet = all ones in both (kBestEmpty; no key reaches it, a
// call holds at most kBestMaxPatterns = 65 535 patterns).  Both updates are commutative, associative and idempotent,
// so the words do not depend on the order of records, passes or chunks, nor on a record reduced twice.
#pragma once
#include "common.cuh"

namespace fzb {

constexpr int kBestThreads = 256;
constexpr uint64_t kBestEmpty = ~0ull;
constexpr uint32_t kBestMaxPatterns = 0xFFFFu;  // ordinals 0 .. 65 534: the all-ones key stays free
constexpr int kBestMaxLen = 2 * kMaxPattern;    // a match is at most len(pattern) + max_l_dist <= 510 long
constexpr uint32_t kBestPairNone = 0xFFFFFFu;

__global__ void k_best_fill(uint64_t *words, uint64_t n) {
    const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) words[i] = kBestEmpty;
}

// `pair` merged into the two smallest pairs with distinct patterns of `word`
__host__ __device__ __forceinline__ uint64_t best_top2_merge(uint64_t word, uint32_t pair) {
    uint32_t first = (uint32_t)(word >> 24) & kBestPairNone, second = (uint32_t)word & kBestPairNone;
    if (pair < first) {
        if ((pair & 0xFFFFu) != (first & 0xFFFFu)) second = first;  // (else: `second` already belongs to another pattern)
        first = pair;
    } else if (pair > first && (pair & 0xFFFFu) != (first & 0xFFFFu) && pair < second) {
        second = pair;
    }
    return 0xFFFF000000000000ull | (uint64_t)first << 24 | second;
}

// One thread per raw record of recs[0..n).  The record of a match is the r with off[r] <= start < off[r + 1], also for
// the empty matches of a pattern with max_l_dist >= its length that sit on the separator closing r (rec_bounds' walk,
// which only reports a separator instead of skipping it).  The pattern is ids[ngram >> 8] for the records of a
// shared pass (MAP), `id` for those of a single search.  Lanes of a warp that hold the same (record, pattern) -- a
// pattern with max_l_dist >= its length emits a record per position -- send one update, the smallest of their keys.
template <bool MAP>
__global__ void k_best_accumulate(const RawRec *recs, uint32_t n, RecSet rs, const uint32_t *ids, uint32_t id,
                                  uint64_t *best, uint64_t *top2) {
    const uint32_t stride = gridDim.x * blockDim.x, lane = threadIdx.x & 31u;
    // (the trip count is the same for the lanes of a warp: the collectives below take all 32)
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; (i & ~31u) < n; i += stride) {
        const bool live = i < n;
        uint64_t key = kBestEmpty, group = kBestEmpty;
        uint32_t r = 0;
        if (live) {
            const RawRec rec = recs[i];
            r = rs.first[rec.start >> kGranuleShift];
            while ((int64_t)rs.off[r + 1] <= rec.start) r++;
            const uint32_t pat = MAP ? ids[(uint32_t)rec.ngram >> 8] : id;
            key = (uint64_t)(uint32_t)rec.dist << 56 | (uint64_t)pat << 40 |
                  (uint64_t)(kBestMaxLen - (rec.end - rec.start)) << 31 | (uint64_t)(rec.start - (int64_t)rs.off[r]);
            group = (uint64_t)r << 16 | pat;
        }
        const unsigned peers = __match_any_sync(0xFFFFFFFFu, group);
        const unsigned shared = __ballot_sync(0xFFFFFFFFu, (peers & (peers - 1)) != 0);  // lanes in groups of 2 or more
        for (unsigned rest = shared; rest; rest &= rest - 1) {
            const int src = __ffs((int)rest) - 1;
            const uint64_t other = __shfl_sync(0xFFFFFFFFu, key, src);
            if (((peers >> src) & 1u) && other < key) key = other;
        }
        if (live && lane == (uint32_t)__ffs((int)peers) - 1u) {
            atomicMin((unsigned long long *)&best[r], (unsigned long long)key);
            const uint32_t pair = (uint32_t)(key >> 40);
            unsigned long long seen = kBestEmpty;  // (a guess: the first match of a record finds it so)
            for (;;) {
                const unsigned long long want = best_top2_merge(seen, pair);
                if (want == seen) break;
                const unsigned long long was = atomicCAS((unsigned long long *)&top2[r], seen, want);
                if (was == seen) break;
                seen = was;
            }
        }
    }
}

}  // namespace fzb
