// common.cuh -- shared declarations for the libfuzzb200 kernels (sm_90a).
#pragma once
#include <cuda.h>
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

// ---- TMA / mbarrier primitives and shared-space loads (sm_90+ PTX) ---------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }

#ifdef FZB_EMU  // tests/emu: mbarrier / TMA semantics restated in C++ (tests/emu/include/cuda.h)
__device__ __forceinline__ void mbar_init(uint64_t *bar, uint32_t count) { emu::mbar_init(bar, count); }
__device__ __forceinline__ void mbar_init_fence() {}
__device__ __forceinline__ void mbar_expect_tx(uint64_t *bar, uint32_t bytes) { emu::mbar_expect_tx(bar, bytes); }
__device__ __forceinline__ void mbar_wait(uint64_t *bar, uint32_t parity) { emu::mbar_wait(bar, parity); }
__device__ __forceinline__ void tma_load_2d(void *dst, const CUtensorMap *map, int c0, int c1, uint64_t *bar) {
    emu::tma_load_2d(dst, map, c0, c1, bar);
}
// cp.async.bulk (1-D): the bytes land, then count against the barrier's expected transaction bytes
__device__ __forceinline__ void bulk_load_1d(void *dst, const void *src, uint32_t bytes, uint64_t *bar) {
    if ((bytes & 15) || ((uintptr_t)src & 15) || (((uintptr_t)dst - (uintptr_t)emu::smem_base()) & 15))
        emu::die("bulk copy: size or address not a multiple of 16");
    memcpy(dst, src, bytes);
    emu::mbar_tx(bar, -(int64_t)bytes, false);
}
#else
__device__ __forceinline__ void mbar_init(uint64_t *bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
// makes the initialised barriers visible to the async proxy (the bulk copies that complete on them)
__device__ __forceinline__ void mbar_init_fence() {
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t *bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t *bar, uint32_t parity) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "WAIT_LOOP:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
        "@p bra WAIT_DONE;\n"
        "bra WAIT_LOOP;\n"
        "WAIT_DONE:\n"
        "}\n" ::"r"(smem_u32(bar)),
        "r"(parity)
        : "memory");
}
__device__ __forceinline__ void tma_load_2d(void *dst, const CUtensorMap *map, int c0, int c1, uint64_t *bar) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];" ::"r"(
            smem_u32(dst)),
        "l"(map), "r"(c0), "r"(c1), "r"(smem_u32(bar))
        : "memory");
}
// contiguous copy of `bytes` (a multiple of 16; src and dst 16-byte aligned) global -> shared, completing on bar
__device__ __forceinline__ void bulk_load_1d(void *dst, const void *src, uint32_t bytes, uint64_t *bar) {
    asm volatile(
        "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(dst)),
        "l"(src), "r"(bytes), "r"(smem_u32(bar))
        : "memory");
}
#endif

// explicit shared-space loads (32-bit shared address: no generic-address arithmetic)
__device__ __forceinline__ uint4 lds128(uint32_t saddr) {
#ifdef FZB_EMU
    return *reinterpret_cast<const uint4 *>(emu::smem_base() + saddr);
#else
    uint4 r;
    asm volatile("ld.shared.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "r"(saddr));
    return r;
#endif
}

__device__ __forceinline__ uint32_t lds32(uint32_t saddr) {
#ifdef FZB_EMU
    return *reinterpret_cast<const uint32_t *>(emu::smem_base() + saddr);
#else
    uint32_t r;
    asm volatile("ld.shared.u32 %0, [%1];" : "=r"(r) : "r"(saddr));
    return r;
#endif
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
