// post_kernels.cuh -- on-device ordering and consolidation of the raw match list (small lists).
//
// ONE kernel runs behind the verify kernel, on the same stream, and replaces the host's sort + sweep for
// lists of up to kPostMax records (the common case: matches are sparse); nothing waits for the host and
// there is no device->host copy operation either: the kernel writes its outputs straight into MAPPED
// pinned host memory, so a search ends with a single stream synchronisation.
//   every CTA  (one per SM) loads the packed canonical keys (start, end-start, dist; written by emit() next to each record) of ALL
//              records into shared memory and ranks its slice of them against all of them (rank = number of
//              smaller keys; a warp ranks two records per pass over the list), scatters its keys to their
//              sorted positions in global memory and takes a ticket.  The all-pairs ranking is spread over every
//              SM rather than run as a single-SM bitonic network or sample sort: one SM issues 4
//              warp-instructions per clock whatever the algorithm.
//   the last   CTA to finish (ticket == grid-1) runs consolidate_overlapping_matches (common.py:145-189) on
//              the sorted keys, one element per thread per round (bank-conflict free): running maximum of
//              `end` as the hull, a record opens a new group iff start >= hull (connected components of
//              interval overlap, SURVEY F11), winner per group = min (dist, -(end-start)), ties -> first in
//              (start, end) order.  Final rows (winner + hull) stay on the device (input of the multi-GPU
//              reduction) and go to the host in coalesced 16-byte stores.
// The raw records themselves stay in device memory; the host fetches them and puts them into the reference's
// generation order lazily, only if a caller asks for the raw stream (api.cu: fetch_raw).
// Larger lists fall back to the host implementation (consolidate_recs in api.cu), which computes
// exactly the same thing.
#pragma once
#include "kernels.cuh"

namespace fzb {

constexpr int kPostMax = 16384;
constexpr int kPostThreads = 1024;
enum { CNT_POST_DONE = 5, CNT_NFINAL = 6, CNT_TICKET = 9, CNT_SEQ = 15 };
constexpr int kFinCols = 5;  // start, end, dist, hull_start, hull_end of the group
constexpr size_t kPostSmem = (size_t)kPostMax * 8 + (size_t)kPostMax * 4;  // keys + per-group best

struct PostArgs {
    const uint64_t *rkeys; // their canonical keys (same order)
    uint32_t cap;          // capacity of recs / rkeys
    int mode;              // 0 raw only; 1 consolidate; 2 final = the raw list in (start, end, dist) order
    uint64_t *sorted;      // device scratch: kPostMax sorted keys
    int64_t *fin;          // device: final rows [kPostMax][kFinCols]
    int64_t *h_fin;        // mapped host: the same rows
    uint32_t *h_counters;  // mapped host: CNT_COUNT counters
    uint32_t *counters;
    uint32_t seq;          // written to h_counters[CNT_SEQ] LAST: the host polls it instead of synchronising the stream
    int clear;             // zero the device counters on the way out (the next search then needs no memset); 0 when
                           // k_push still has to read them
};

__device__ __forceinline__ uint32_t gtimer_lo() {
#ifdef FZB_EMU
    return (uint32_t)emu::cycles();
#else
    unsigned long long t;
    asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t));
    return (uint32_t)t;
#endif
}

// Block-wide exclusive scans of one value per thread (1024 threads = 32 warps); *total = sum / max of all.
// scratch: 33 entries.
__device__ __forceinline__ uint32_t block_scan_sum(uint32_t v, uint32_t *scratch, uint32_t *total) {
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    uint32_t inc = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const uint32_t t = __shfl_up_sync(0xFFFFFFFFu, inc, o);
        if (lane >= o) inc += t;
    }
    if (lane == 31) scratch[w] = inc;
    __syncthreads();
    if (w == 0) {
        const uint32_t x = scratch[lane];
        uint32_t xi = x;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const uint32_t t = __shfl_up_sync(0xFFFFFFFFu, xi, o);
            if (lane >= o) xi += t;
        }
        scratch[lane] = xi - x;  // exclusive
        if (lane == 31) scratch[32] = xi;
    }
    __syncthreads();
    const uint32_t r = scratch[w] + inc - v;
    *total = scratch[32];
    __syncthreads();
    return r;
}

__device__ __forceinline__ unsigned long long block_scan_max(unsigned long long v, unsigned long long *scratch,
                                                             unsigned long long *total) {
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    unsigned long long inc = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const unsigned long long t = __shfl_up_sync(0xFFFFFFFFu, inc, o);
        if (lane >= o) inc = max(inc, t);
    }
    unsigned long long exc = __shfl_up_sync(0xFFFFFFFFu, inc, 1);
    if (lane == 0) exc = 0;
    if (lane == 31) scratch[w] = inc;
    __syncthreads();
    if (w == 0) {
        const unsigned long long x = scratch[lane];
        unsigned long long xi = x;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const unsigned long long t = __shfl_up_sync(0xFFFFFFFFu, xi, o);
            if (lane >= o) xi = max(xi, t);
        }
        unsigned long long xe = __shfl_up_sync(0xFFFFFFFFu, xi, 1);
        if (lane == 0) xe = 0;
        scratch[lane] = xe;  // exclusive
        if (lane == 31) scratch[32] = xi;
    }
    __syncthreads();
    const unsigned long long r = max(scratch[w], exc);
    *total = scratch[32];
    __syncthreads();
    return r;
}

__global__ void __launch_bounds__(kPostThreads, 1)
k_post(const PostArgs a) {
    extern __shared__ __align__(16) uint8_t post_smem[];
    uint64_t *keys = reinterpret_cast<uint64_t *>(post_smem);
    uint32_t *segbest = reinterpret_cast<uint32_t *>(post_smem + (size_t)kPostMax * 8);
    __shared__ unsigned long long scr64[33];
    __shared__ uint32_t scr32[33];
    __shared__ uint32_t s_ticket;
    const uint32_t nraw = a.counters[CNT_OUT];
    const uint32_t n = a.counters[CNT_KEYS];  // distinct-ish keys (<= nraw): what gets ordered and consolidated
    const bool fits = nraw <= (uint32_t)kPostMax && nraw <= a.cap;
    const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const uint32_t G = gridDim.x, b = blockIdx.x;
    if (!fits) {  // the host fetches the list and does the rest
        if (b == 0) {
            if (tid < CNT_SEQ) a.h_counters[tid] = a.counters[tid];  // POST_DONE stays 0 (and the counters stay dirty:
            __threadfence_system();                                   //  other CTAs may not have read them yet)
            __syncthreads();
            if (tid == 0) a.h_counters[CNT_SEQ] = a.seq;
        }
        return;
    }
    const uint32_t t_start = gtimer_lo();
    const uint32_t lo = (uint32_t)((uint64_t)n * b / G), hi = (uint32_t)((uint64_t)n * (b + 1) / G);
    if (a.mode != 0 && n > 0) {
        for (uint32_t i = tid; i < n; i += kPostThreads) keys[i] = a.rkeys[i];
        __syncthreads();
        // rank: a warp takes two records of my slice per pass, its lanes split the list
        for (uint32_t i0 = lo + 2 * warp; i0 < hi; i0 += 2 * (kPostThreads / 32)) {
            const uint32_t i1 = min(i0 + 1, hi - 1);
            const uint64_t key0 = keys[i0], key1 = keys[i1];
            uint32_t c0 = 0, c1 = 0;
            for (uint32_t j = lane; j < n; j += 32) {
                const uint64_t kj = keys[j];
                c0 += (kj < key0) || (kj == key0 && j < i0);
                c1 += (kj < key1) || (kj == key1 && j < i1);
            }
            c0 = __reduce_add_sync(0xFFFFFFFFu, c0);
            c1 = __reduce_add_sync(0xFFFFFFFFu, c1);
            if (lane == 0) {
                a.sorted[c0] = key0;
                a.sorted[c1] = key1;  // (i1 == i0 for an odd tail: the same store twice)
            }
        }
    }
    const uint32_t t_ranked = gtimer_lo();
    __threadfence();
    __syncthreads();
    if (tid == 0) s_ticket = atomicAdd(&a.counters[CNT_TICKET], 1u);
    __syncthreads();
    if (s_ticket != G - 1) return;
    __threadfence();  // every other CTA's scatter is visible now
    const uint32_t t_ticket = gtimer_lo();
    uint32_t t_sorted = t_ticket, t_swept = t_ticket;
    uint32_t nfinal = 0;
    if (a.mode != 0 && n > 0) {
        for (uint32_t i = tid; i < n; i += kPostThreads) keys[i] = __ldcg(a.sorted + i);
        __syncthreads();
        t_sorted = gtimer_lo();
        // ---- final rows --------------------------------------------------------------------------
        if (a.mode == 2) {  // unconsolidated routes: the final list is the sorted raw list
            nfinal = n;
            for (uint32_t i = tid; i < n; i += kPostThreads) {
                const uint64_t kx = keys[i];
                const int64_t s = (int64_t)(kx >> 18), e = s + (int64_t)((kx >> 8) & 1023u);
                int64_t *row = a.fin + (size_t)kFinCols * i;
                row[0] = s;
                row[1] = e;
                row[2] = (int64_t)(kx & 255u);
                row[3] = s;
                row[4] = e;
            }
        } else {
            for (uint32_t i = tid; i < n; i += kPostThreads) segbest[i] = 0xFFFFFFFFu;
            __syncthreads();
            unsigned long long carry_hull = 0;  // max end of all earlier rounds
            uint32_t carry_groups = 0;          // groups opened in earlier rounds
            for (uint32_t base = 0; base < n; base += kPostThreads) {
                const uint32_t i = base + tid;
                const bool live = i < n;
                const uint64_t kx = live ? keys[i] : 0;
                const unsigned long long s = kx >> 18, len = (kx >> 8) & 1023u, e = live ? s + len : 0;
                unsigned long long round_max;
                const unsigned long long hull = max(carry_hull, block_scan_max(e, scr64, &round_max));  // exclusive
                const bool head = live && (i == 0 || s >= hull);
                uint32_t round_heads;
                const uint32_t before = block_scan_sum(head ? 1u : 0u, scr32, &round_heads);
                if (live) {
                    const uint32_t g = carry_groups + before + (head ? 1u : 0u) - 1u;  // my group
                    if (head) {
                        a.fin[(size_t)kFinCols * g + 3] = (int64_t)s;                       // hull start of my group
                        if (g >= 1) a.fin[(size_t)kFinCols * (g - 1) + 4] = (int64_t)hull;  // hull end of the previous
                    }
                    if (i == n - 1) a.fin[(size_t)kFinCols * g + 4] = (int64_t)max(hull, e);  // last group
                    const uint32_t score = ((uint32_t)(kx & 255u) << 24) | ((uint32_t)(1023u - len) << 14) | i;
                    atomicMin(&segbest[g], score);
                }
                carry_hull = max(carry_hull, round_max);
                carry_groups += round_heads;
            }
            nfinal = carry_groups;
            __syncthreads();
            for (uint32_t g = tid; g < nfinal; g += kPostThreads) {
                const uint64_t kx = keys[segbest[g] & 16383u];
                const int64_t s = (int64_t)(kx >> 18);
                int64_t *row = a.fin + (size_t)kFinCols * g;
                row[0] = s;
                row[1] = s + (int64_t)((kx >> 8) & 1023u);
                row[2] = (int64_t)(kx & 255u);
            }
        }
        // device rows -> host, coalesced 16-byte stores (rows are 40 bytes: copy the whole block as uint4)
        __threadfence_block();
        __syncthreads();
        t_swept = gtimer_lo();
        const uint32_t nvec = (uint32_t)(((size_t)nfinal * kFinCols * 8 + 15) / 16);
        const uint4 *src = reinterpret_cast<const uint4 *>(a.fin);
        uint4 *dst = reinterpret_cast<uint4 *>(a.h_fin);
        for (uint32_t i = tid; i < nvec; i += kPostThreads) dst[i] = __ldcg(src + i);
    }
    __syncthreads();
    if (tid == 0) {
        a.counters[CNT_NFINAL] = nfinal;
        a.counters[CNT_POST_DONE] = 1u;
        // phase times of the last CTA in ns (fzb_debug_counters): copy + rank, ticket + reload, sweep, copy-out
        a.counters[10] = t_ranked - t_start;
        a.counters[11] = t_sorted - t_ranked;
        a.counters[12] = t_swept - t_sorted;
        a.counters[13] = gtimer_lo() - t_swept;
    }
    __syncthreads();
    if (tid < CNT_SEQ) a.h_counters[tid] = a.counters[tid];
    if (a.clear && tid < CNT_COUNT) a.counters[tid] = 0;
    __threadfence_system();
    __syncthreads();
    if (tid == 0) a.h_counters[CNT_SEQ] = a.seq;  // everything above is visible to the host before this word
}

}  // namespace fzb
