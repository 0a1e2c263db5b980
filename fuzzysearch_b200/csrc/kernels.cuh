// kernels.cuh -- sm_90a kernels of libfuzzb200 (Levenshtein n-gram route, exact search, Hamming).
//
// Pipeline of one n-gram search (DESIGN.md section 3):
//   k_filter_sampled / k_filter_dense : ONE pass over the haystack (the HBM-bound kernel); marks
//        64-position "granules" that may contain an n-gram hit of a <=k-error occurrence.
//   k_verify_lev : re-examines only the marked granules: exact n-gram test at every position,
//        then the reference's right/left expansion DP per hit; emits raw (start,end,dist) triples.
#pragma once
#include "common.cuh"

namespace fzb {

// ------------------------------------------------------------------------------------------------
// small helpers
// ------------------------------------------------------------------------------------------------
constexpr int kTblBits = 15;                   // hashed byte table: 32 KiB of shared memory
constexpr int kTblSize = 1 << kTblBits;
constexpr uint32_t kHashMul = 0x9E3779B1u;
constexpr int kFilterThreads = 256;
constexpr int kFilterUnroll = 4;               // uint4 loads in flight per thread
constexpr int kTileVecs = kFilterThreads * kFilterUnroll;  // uint4s per CTA tile (16 KiB)

__device__ __forceinline__ uint32_t hash_word(uint32_t w) { return (w * kHashMul) >> (32 - kTblBits); }

__device__ __forceinline__ uint4 ldg_stream(const uint4 *p) {
#ifdef FZB_EMU  // tests/emu: the CPU replay of these sources has no PTX
    return *p;
#else
    uint4 r;
    asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
                 : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
                 : "l"(p));
    return r;
#endif
}

// Mark granule g.  The bitmap de-duplicates; the thread that flips the bit 0 -> 1 also appends the
// granule to the verify kernel's work list (no separate compaction pass over the bitmap).  If the list
// is full the bit simply stays set and the verify kernel's bitmap sweep picks it up.
__device__ __forceinline__ void mark_granule(uint32_t *bitmap, uint32_t *glist, uint32_t glist_cap,
                                             uint32_t *counters, int64_t g) {
    const uint32_t bit = 1u << (g & 31);
    const uint32_t old = atomicOr(&bitmap[g >> 5], bit);
    if (!(old & bit)) {
        const uint32_t slot = atomicAdd(&counters[CNT_GRAN], 1u);
        if (slot < glist_cap) glist[slot] = (uint32_t)g;
    }
}

// The few scalars marking needs, passed BY VALUE to the out-of-line slow paths (a reference to the
// kernel's ScanParams would force a local-memory copy of the whole parameter block, and inlining the
// atomics into the streaming loops upsets their register allocation).
struct MarkCtx {
    int64_t buf_lo, own_lo, own_hi;
    uint32_t *bitmap;
    uint32_t *glist;
    uint32_t glist_cap;
    uint64_t *hits;
    uint32_t hits_cap;
    uint32_t *counters;
};

__device__ __forceinline__ MarkCtx mark_ctx(const ScanParams &p) {
    return MarkCtx{p.buf_lo, p.own_lo, p.own_hi, p.bitmap, p.glist, p.glist_cap, p.hits, p.hits_cap, p.counters};
}

// mark the granules covering anchors [lo, hi] (global coords), clipped to the owned range
__device__ __noinline__ void mark_range_ctx(MarkCtx mc, int64_t lo, int64_t hi) {
    if (lo < mc.own_lo) lo = mc.own_lo;
    if (hi > mc.own_hi - 1) hi = mc.own_hi - 1;
    if (lo > hi) return;
    int64_t g0 = (lo - mc.buf_lo) >> kGranuleShift, g1 = (hi - mc.buf_lo) >> kGranuleShift;
    for (int64_t g = g0; g <= g1; g++) mark_granule(mc.bitmap, mc.glist, mc.glist_cap, mc.counters, g);
}

__device__ __forceinline__ void mark_range(const ScanParams &p, int64_t lo, int64_t hi) {
    mark_range_ctx(mark_ctx(p), lo, hi);
}

// inlined variant for kernels whose register budget is pinned anyway (k_hamming_count)
__device__ __forceinline__ void mark_range_inline(const ScanParams &p, int64_t lo, int64_t hi) {
    if (lo < p.own_lo) lo = p.own_lo;
    if (hi > p.own_hi - 1) hi = p.own_hi - 1;
    if (lo > hi) return;
    int64_t g0 = (lo - p.buf_lo) >> kGranuleShift, g1 = (hi - p.buf_lo) >> kGranuleShift;
    for (int64_t g = g0; g <= g1; g++) mark_granule(p.bitmap, p.glist, p.glist_cap, p.counters, g);
}

// ------------------------------------------------------------------------------------------------
// Sampled filter (stride 4).  Soundness (q-sample lemma): a raw match (start,end,dist<=k) of the
// n-gram search spans an occurrence O=H[start:end] with ED(P,O)<=k and |O|>=m-k.  O contains at
// least floor((m-k-3)/4) 4-byte-aligned words; k edits touch at most k of them; the host selects
// this kernel only if floor((m-k-3)/4) >= k+1, so at least one aligned word inside O equals some
// 4-gram of P.  Each aligned word is looked up (multiplicative hash -> byte table in shared
// memory); table hits are re-checked exactly against the pattern's 4-grams and then mark every
// granule that can hold an n-gram anchor of an occurrence containing that word.
// Per 4 haystack bytes: IMAD (hash) + SHF + LDS.U8 + IMAD (accumulate): ~1 issue slot per byte.
// ------------------------------------------------------------------------------------------------
// Confirmation of table hits is warp-cooperative and branch-uniform: the flagged lane's word is
// broadcast and lane o compares it with the pattern's o-th 4-gram (one compare per lane), so the
// common case (no lane flagged: one ballot) and the rare case (a false positive of the hash) both
// cost a handful of warp instructions and nothing is spilled to local memory.
__device__ __forceinline__ void confirm_word(const ScanParams &p, const uint32_t *grams, int ngr, int lane,
                                             uint32_t w, int64_t word_off) {
    bool real = false;
    for (int o = lane; o < ngr; o += 32) real |= (grams[o] == w);
    if (__ballot_sync(0xFFFFFFFFu, real) != 0 && lane == 0) {
        const int64_t g = p.buf_lo + word_off;
        // anchor idx of n-gram j (pattern offset s_j in [0, m-L]) of an occurrence containing the
        // word:  idx - s_j - k <= g  and  g + 4 <= idx - s_j + m + k
        mark_range(p, g - (p.m + p.k - 4), g + (p.m - p.L + p.k));
    }
}

__global__ void __launch_bounds__(kFilterThreads)
k_filter_sampled(const ScanParams p, int64_t nvec, int64_t ntiles) {
    extern __shared__ __align__(16) uint8_t smem[];
    uint8_t *tbl = smem;
    uint32_t *grams = reinterpret_cast<uint32_t *>(smem + kTblSize);
    for (int i = threadIdx.x; i < kTblSize / 16; i += blockDim.x)
        reinterpret_cast<uint4 *>(tbl)[i] = make_uint4(0, 0, 0, 0);
    __syncthreads();
    const int ngr = p.m - 3;
    for (int o = threadIdx.x; o < ngr; o += blockDim.x) {
        uint32_t w = (uint32_t)p.P[o] | ((uint32_t)p.P[o + 1] << 8) | ((uint32_t)p.P[o + 2] << 16) |
                     ((uint32_t)p.P[o + 3] << 24);
        grams[o] = w;
        tbl[hash_word(w)] = 1;
    }
    __syncthreads();

    const int lane = threadIdx.x & 31;
    const uint4 *base = reinterpret_cast<const uint4 *>(p.H);
    for (int64_t t = blockIdx.x; t < ntiles; t += gridDim.x) {
        const int64_t v0 = t * kTileVecs + threadIdx.x;
        uint4 d[kFilterUnroll];
#pragma unroll
        for (int u = 0; u < kFilterUnroll; u++) {
            int64_t v = v0 + (int64_t)u * kFilterThreads;
            d[u] = (v < nvec) ? ldg_stream(base + v) : make_uint4(0, 0, 0, 0);
        }
        uint32_t acc = 0;  // bit (4*kFilterUnroll - 1 - 4u - i) <-> word i of load u
#pragma unroll
        for (int u = 0; u < kFilterUnroll; u++) {
            acc = acc * 2u + tbl[hash_word(d[u].x)];
            acc = acc * 2u + tbl[hash_word(d[u].y)];
            acc = acc * 2u + tbl[hash_word(d[u].z)];
            acc = acc * 2u + tbl[hash_word(d[u].w)];
        }
        unsigned flagged = __ballot_sync(0xFFFFFFFFu, acc != 0);
        while (flagged) {  // warp-uniform
            const int src = __ffs(flagged) - 1;
            flagged &= flagged - 1;
            const uint32_t a = __shfl_sync(0xFFFFFFFFu, acc, src);
            const int64_t vsrc = t * kTileVecs + (threadIdx.x - lane + src);
#pragma unroll
            for (int u = 0; u < kFilterUnroll; u++) {
                if ((a >> (4 * (kFilterUnroll - 1 - u))) & 0xFu) {  // uniform
                    const int64_t off = (vsrc + (int64_t)u * kFilterThreads) * 16;
                    const uint32_t wx = __shfl_sync(0xFFFFFFFFu, d[u].x, src);
                    const uint32_t wy = __shfl_sync(0xFFFFFFFFu, d[u].y, src);
                    const uint32_t wz = __shfl_sync(0xFFFFFFFFu, d[u].z, src);
                    const uint32_t ww = __shfl_sync(0xFFFFFFFFu, d[u].w, src);
                    const uint32_t nib = a >> (4 * (kFilterUnroll - 1 - u));
                    if (nib & 8u) confirm_word(p, grams, ngr, lane, wx, off);
                    if (nib & 4u) confirm_word(p, grams, ngr, lane, wy, off + 4);
                    if (nib & 2u) confirm_word(p, grams, ngr, lane, wz, off + 8);
                    if (nib & 1u) confirm_word(p, grams, ngr, lane, ww, off + 12);
                }
            }
        }
    }
}

// ------------------------------------------------------------------------------------------------
// Dense filter (every position): used when the q-sample lemma does not apply (short patterns / large
// k) or when it is not selective (small alphabets: on DNA an aligned 4-byte word carries 8 bits and
// almost every granule would be marked).  It tests the first q = min(L, 8) bytes at EVERY position
// against the n-grams themselves, i.e. it finds the n-gram hits of levenshtein_ngram.py:176 directly:
//   per position: two funnel shifts build the 8-byte window (lo, hi), a 2-multiply hash picks one bit
//   of an 8 Kibit table, replicated once per shared-memory bank so that lane l always reads bank l
//   (address = row * 128 + 4 l: every lookup is one conflict-free wavefront).
// Hits are confirmed warp-cooperatively (ballot, broadcast the window, lane j compares with n-gram j)
// and mark the granule of that anchor position only.
// ------------------------------------------------------------------------------------------------
constexpr int kDenseBits = 13;                       // 8 Kibit table ...
constexpr int kDenseRows = (1 << kDenseBits) / 32;   // ... = 256 rows of 32 bits, one copy per bank
constexpr int kDenseWarpScratch = 8 + 2 + 64;      // words per warp: 6-word window, count, 32 buffered hits (u64)
constexpr size_t kDenseSmem = (size_t)kDenseRows * 128 + 256 * 8 + 8 * kDenseWarpScratch * 4;  // 32 KiB + windows + scratch
constexpr uint32_t kHashMul2 = 0x85EBCA77u;

__device__ __forceinline__ uint32_t dense_key(uint32_t lo, uint32_t hi) {
    return (lo * kHashMul + hi * kHashMul2) >> (32 - kDenseBits);
}

// Flush the warp's buffered hits to the global hit list (one atomicAdd for all of them).
__device__ __forceinline__ void dense_flush_hits(const MarkCtx &mc, uint32_t *scratch, int lane) {
    __syncwarp();
    const uint32_t n = scratch[8];
    if (n == 0) return;
    uint32_t base = 0;
    if (lane == 0) base = atomicAdd(&mc.counters[CNT_HITS], n);
    base = __shfl_sync(0xFFFFFFFFu, base, 0);
    const uint64_t *buf = reinterpret_cast<const uint64_t *>(scratch + 10);
    if ((uint32_t)lane < n && base + lane < mc.hits_cap) mc.hits[base + lane] = buf[lane];
    __syncwarp();
    if (lane == 0) scratch[8] = 0;
    __syncwarp();
}

// Slow path of the dense filter, for the whole warp: every flagged lane in turn parks its six words in
// a per-warp scratch line, then all lanes walk its set bits, rebuild the 8-byte window at that byte
// offset from the scratch and lane j compares it with n-gram j.
__device__ __noinline__ void dense_confirm_warp(MarkCtx mc, int n_ngrams, const uint2 *grams, uint32_t *scratch,
                                                int lane, unsigned flagged, uint32_t acc, uint32_t w0_, uint32_t w1_,
                                                uint32_t w2_, uint32_t w3_, uint32_t w4_, uint32_t w5_,
                                                int64_t off_warp, uint32_t mlo, uint32_t mhi) {
    while (flagged) {
        const int src = __ffs(flagged) - 1;
        flagged &= flagged - 1;
        uint32_t a = __shfl_sync(0xFFFFFFFFu, acc, src);
        __syncwarp();
        if (lane == src) {
            scratch[0] = w0_;
            scratch[1] = w1_;
            scratch[2] = w2_;
            scratch[3] = w3_;
            scratch[4] = w4_;
            scratch[5] = w5_;
        }
        __syncwarp();
        while (a) {
            const int bit = 31 - __clz(a);  // bit 15 <-> byte 0
            a &= ~(1u << bit);
            const int b = 15 - bit;
            const uint32_t w0 = scratch[b >> 2], w1 = scratch[(b >> 2) + 1], w2 = scratch[(b >> 2) + 2];
            const uint32_t lo = __funnelshift_r(w0, w1, 8 * (b & 3)) & mlo;
            const uint32_t hi = __funnelshift_r(w1, w2, 8 * (b & 3)) & mhi;
            const int64_t g = mc.buf_lo + off_warp + (int64_t)src * 16 + b;
            const bool owned = g >= mc.own_lo && g < mc.own_hi;
            if (mc.hits_cap) {  // hit-list mode: one entry per (n-gram, position); verified lane-parallel later
                // hits are buffered per warp in shared memory and flushed 24+ at a time: one global
                // atomic per flush instead of one per hit (millions of hits on low-entropy data)
                uint32_t &cnt = scratch[8];
                uint64_t *buf = reinterpret_cast<uint64_t *>(scratch + 10);
                for (int j0 = 0; j0 < n_ngrams; j0 += 32) {
                    const int j = j0 + lane;
                    const bool mt = owned && j < n_ngrams && grams[j].x == lo && grams[j].y == hi;
                    const unsigned bm = __ballot_sync(0xFFFFFFFFu, mt);
                    if (!bm) continue;
                    uint32_t c0 = cnt;
                    if (c0 + __popc(bm) > 32) {  // make room first
                        dense_flush_hits(mc, scratch, lane);
                        c0 = 0;
                    }
                    if (mt) buf[c0 + __popc(bm & ((1u << lane) - 1u))] = ((uint64_t)g << 8) | (uint64_t)j;
                    __syncwarp();
                    if (lane == 0) cnt = c0 + __popc(bm);
                    __syncwarp();
                }
            } else {
                bool real = false;
                for (int j = lane; j < n_ngrams; j += 32) real |= (grams[j].x == lo && grams[j].y == hi);
                if (__ballot_sync(0xFFFFFFFFu, real) != 0 && lane == 0 && owned) {
                    mark_granule(mc.bitmap, mc.glist, mc.glist_cap, mc.counters, (g - mc.buf_lo) >> kGranuleShift);
                }
            }
        }
    }
    if (mc.hits_cap && scratch[8] >= 24) dense_flush_hits(mc, scratch, lane);
}

// MODE: 0 = q < 4 (lo masked), 1 = q == 4, 2 = 4 < q < 8 (hi masked), 3 = q == 8 -- compile-time so that the
// short-n-gram cases do not pay for the second funnel shift, the masks and the second multiply.
template <int MODE>
__global__ void __launch_bounds__(kFilterThreads)
k_filter_dense(const ScanParams p, int64_t nvec, int64_t ntiles) {
    extern __shared__ __align__(16) uint8_t smem[];
    uint32_t *tbl = reinterpret_cast<uint32_t *>(smem);                        // [kDenseRows][32 banks]
    uint2 *grams = reinterpret_cast<uint2 *>(smem + (size_t)kDenseRows * 128);  // (lo, hi) per n-gram (<= 255)
    uint32_t *scratch = reinterpret_cast<uint32_t *>(smem + (size_t)kDenseRows * 128 + 256 * 8) +
                        (threadIdx.x >> 5) * kDenseWarpScratch;  // this warp's window / hit buffer
    if ((threadIdx.x & 31) == 0) scratch[8] = 0;
    for (int i = threadIdx.x; i < kDenseRows * 32 / 4; i += blockDim.x)
        reinterpret_cast<uint4 *>(tbl)[i] = make_uint4(0, 0, 0, 0);
    __syncthreads();
    const int q = p.q;  // 1..8
    const uint32_t mlo = q >= 4 ? 0xFFFFFFFFu : ((1u << (8 * q)) - 1u);
    const uint32_t mhi = q <= 4 ? 0u : (q >= 8 ? 0xFFFFFFFFu : ((1u << (8 * (q - 4))) - 1u));
    if (threadIdx.x < 32) {  // lane l fills its own bank's copy (the n-gram count is small)
        for (int j = 0; j < p.n_ngrams; j++) {
            uint32_t lo = 0, hi = 0;
            for (int b = 0; b < q; b++) {
                const uint32_t c = p.P[j * p.L + b];
                if (b < 4) lo |= c << (8 * b); else hi |= c << (8 * (b - 4));
            }
            if (threadIdx.x == 0) grams[j] = make_uint2(lo, hi);
            const uint32_t key = dense_key(lo, hi);
            tbl[(key >> 5) * 32 + threadIdx.x] |= 1u << (key & 31);
        }
    }
    __syncthreads();

    const int lane = threadIdx.x & 31;
    const uint32_t my_bank = (uint32_t)__cvta_generic_to_shared(tbl) + 4u * lane;
    const uint4 *base = reinterpret_cast<const uint4 *>(p.H);
    for (int64_t t = blockIdx.x; t < ntiles; t += gridDim.x) {
        const int64_t v0 = t * kTileVecs + threadIdx.x;
        // two loads in flight per thread (memory-level parallelism), then the per-position work
#pragma unroll 1
        for (int uh = 0; uh < kFilterUnroll; uh += 2) {
        uint4 dd[2];
        uint2 nn[2];
#pragma unroll
        for (int u2 = 0; u2 < 2; u2++) {
            const int64_t v = v0 + (int64_t)(uh + u2) * kFilterThreads;
            dd[u2] = (v < nvec) ? ldg_stream(base + v) : make_uint4(0, 0, 0, 0);
            nn[u2] = make_uint2(0, 0);
            // the 8 bytes after my 16: the neighbour lane has them, the last lane reads them itself
            if (lane == 31 && v < nvec) nn[u2] = __ldg(reinterpret_cast<const uint2 *>(base + v + 1));  // padded buffer
        }
#pragma unroll
        for (int u2 = 0; u2 < 2; u2++) {
            const int u = uh + u2;
            const uint4 d = dd[u2];
            uint32_t n0 = __shfl_down_sync(0xFFFFFFFFu, d.x, 1), n1 = __shfl_down_sync(0xFFFFFFFFu, d.y, 1);
            if (lane == 31) {
                n0 = nn[u2].x;
                n1 = nn[u2].y;
            }
            const uint32_t ws[6] = {d.x, d.y, d.z, d.w, n0, n1};
            uint32_t acc = 0;
#pragma unroll
            for (int b = 0; b < 16; b++) {
                uint32_t lo = __funnelshift_r(ws[b >> 2], ws[(b >> 2) + 1], 8 * (b & 3));
                if (MODE == 0) lo &= mlo;
                uint32_t key;
                if (MODE <= 1) {
                    key = (lo * kHashMul) >> (32 - kDenseBits);  // == dense_key(lo, 0)
                } else {
                    uint32_t hi = __funnelshift_r(ws[(b >> 2) + 1], ws[(b >> 2) + 2], 8 * (b & 3));
                    if (MODE == 2) hi &= mhi;
                    key = dense_key(lo, hi);
                }
                uint32_t row;
#ifdef FZB_EMU
                row = *reinterpret_cast<const uint32_t *>(emu::smem_base() + my_bank + ((key >> 5) << 7));
#else
                asm volatile("ld.shared.u32 %0, [%1];" : "=r"(row) : "r"(my_bank + ((key >> 5) << 7)));
#endif
                acc = acc * 2u + (__funnelshift_r(row, 0u, key) & 1u);  // bit (key & 31) of the row
            }
            unsigned flagged = __ballot_sync(0xFFFFFFFFu, acc != 0);
            if (flagged) {  // warp-uniform, kept out of line and compact (instruction cache)
                const int64_t off_warp = (t * kTileVecs + (threadIdx.x - lane) + (int64_t)u * kFilterThreads) * 16;
                dense_confirm_warp(mark_ctx(p),
                                   p.n_ngrams, grams,
                                   scratch, lane, flagged, acc, ws[0], ws[1], ws[2], ws[3],
                                   ws[4], ws[5], off_warp, mlo, mhi);
            }
        }
        }
    }
    if (p.hits_cap) dense_flush_hits(mark_ctx(p), scratch, lane);  // what is still buffered
}

// ------------------------------------------------------------------------------------------------
// Dense filter for LOW-ENTROPY haystacks (DNA and the like), where the dense route actually runs.  The text is
// reduced to 2-bit codes, code(c) = (c >> 1) & 3 -- distinct for A, C, G, T; any other byte merely aliases with one
// of them, which can only add candidates (the confirmation compares the real bytes).  A lane packs its 16 bytes into
// one 32-bit word (one multiply per 4 bytes) and fetches 8 more codes from its neighbour; then ONE table lookup
// answers THREE positions: the table is indexed by 8 consecutive codes (16 bits, 64 KiB of bytes in shared memory)
// and entry bit i says whether the min(L,6)-code window starting at code i is the prefix of some n-gram.  Six
// lookups per 16 positions: ~4 thread-instructions per position where the hashing k_filter_dense spends ~19.
// Table hits are confirmed by the flagged lane itself against the n-grams' real bytes (a few dozen instructions
// per hit, several flagged lanes run side by side) and go to the warp's hit buffer / the granule bitmap as in
// k_filter_dense.
// ------------------------------------------------------------------------------------------------
constexpr int kD2Bases = 6;                   // codes of an n-gram the table looks at
constexpr int kD2Span = 8;                    // codes per table index: three windows of six
constexpr size_t kDense2Smem = (size_t)(1 << (2 * kD2Span)) + 256 * 8 + 8 * kDenseWarpScratch * 4;

__host__ __device__ __forceinline__ uint32_t pack2(uint32_t w) {  // 4 bytes -> 4 two-bit codes in bits 0..7
    return (((w >> 1) & 0x03030303u) * 0x01041040u) >> 24;
}

__global__ void __launch_bounds__(kFilterThreads, 3)
k_filter_dense2(const ScanParams p, int64_t nvec, int64_t ntiles) {
    extern __shared__ __align__(16) uint8_t smem[];
    uint8_t *tbl = smem;                                                          // [65536] bits 0..2
    uint2 *grams = reinterpret_cast<uint2 *>(smem + (1 << (2 * kD2Span)));       // (lo, hi) per n-gram (<= 255)
    uint32_t *scratch = reinterpret_cast<uint32_t *>(smem + (1 << (2 * kD2Span)) + 256 * 8) +
                        (threadIdx.x >> 5) * kDenseWarpScratch;                   // this warp's hit buffer
    if ((threadIdx.x & 31) == 0) scratch[8] = 0;
    for (int i = threadIdx.x; i < (1 << (2 * kD2Span)) / 16; i += blockDim.x)
        reinterpret_cast<uint4 *>(tbl)[i] = make_uint4(0, 0, 0, 0);
    __syncthreads();
    const int q = p.q;  // 1..8 raw bytes compared by the confirmation
    const int qc = min(q, kD2Bases);
    const uint32_t cmask = (1u << (2 * qc)) - 1u;
    const uint32_t mlo = q >= 4 ? 0xFFFFFFFFu : ((1u << (8 * q)) - 1u);
    const uint32_t mhi = q <= 4 ? 0u : (q >= 8 ? 0xFFFFFFFFu : ((1u << (8 * (q - 4))) - 1u));
    __shared__ uint32_t sSet[128];  // 4096-bit set of the n-grams' code prefixes (build phase only)
    for (int i = threadIdx.x; i < 128; i += blockDim.x) sSet[i] = 0;
    __syncthreads();
    if (threadIdx.x == 0) {
        for (int j = 0; j < p.n_ngrams; j++) {
            uint32_t lo = 0, hi = 0, code = 0;
            for (int b = 0; b < q; b++) {
                const uint32_t c = p.P[j * p.L + b];
                if (b < 4) lo |= c << (8 * b); else hi |= c << (8 * (b - 4));
                if (b < qc) code |= ((c >> 1) & 3u) << (2 * b);
            }
            grams[j] = make_uint2(lo, hi);
            sSet[code >> 5] |= 1u << (code & 31);
        }
    }
    __syncthreads();
    for (uint32_t e = threadIdx.x; e < (1u << (2 * kD2Span)); e += blockDim.x) {
        uint32_t v = 0;
#pragma unroll
        for (int i = 0; i < 3; i++) {
            const uint32_t c = (e >> (2 * i)) & cmask;
            v |= ((sSet[c >> 5] >> (c & 31)) & 1u) << i;
        }
        tbl[e] = (uint8_t)v;
    }
    __syncthreads();

    const int lane = threadIdx.x & 31;
    const MarkCtx mc = mark_ctx(p);
    unsigned long long *hbuf = reinterpret_cast<unsigned long long *>(scratch + 10);
    const uint4 *base = reinterpret_cast<const uint4 *>(p.H);
    for (int64_t t = blockIdx.x; t < ntiles; t += gridDim.x) {
        const int64_t v0 = t * kTileVecs + threadIdx.x;
#pragma unroll 1
        for (int uh = 0; uh < kFilterUnroll; uh += 2) {
        uint4 dd[2];
        uint2 nn[2];
#pragma unroll
        for (int u2 = 0; u2 < 2; u2++) {
            const int64_t v = v0 + (int64_t)(uh + u2) * kFilterThreads;
            dd[u2] = (v < nvec) ? ldg_stream(base + v) : make_uint4(0, 0, 0, 0);
            nn[u2] = make_uint2(0, 0);
            if (lane == 31 && v < nvec) nn[u2] = __ldg(reinterpret_cast<const uint2 *>(base + v + 1));  // padded buffer
        }
#pragma unroll
        for (int u2 = 0; u2 < 2; u2++) {
            const int u = uh + u2;
            const uint4 d = dd[u2];
            uint32_t n0 = __shfl_down_sync(0xFFFFFFFFu, d.x, 1), n1 = __shfl_down_sync(0xFFFFFFFFu, d.y, 1);
            if (lane == 31) {
                n0 = nn[u2].x;
                n1 = nn[u2].y;
            }
            const uint32_t pk = pack2(d.x) | (pack2(d.y) << 8) | (pack2(d.z) << 16) | (pack2(d.w) << 24);
            const uint32_t nx = pack2(n0) | (pack2(n1) << 8);
            uint32_t acc = 0;  // bit i <-> position i of my vector
#pragma unroll
            for (int g3 = 0; g3 < 6; g3++)  // positions 3*g3 .. 3*g3+2 (the last lookup's bits 16, 17 are dropped)
                acc |= (uint32_t)tbl[__funnelshift_r(pk, nx, 6 * g3) & 0xFFFFu] << (3 * g3);
            acc &= 0xFFFFu;
            if (acc) {  // rare; flagged lanes confirm their own positions side by side
                const int64_t off = (t * kTileVecs + threadIdx.x + (int64_t)u * kFilterThreads) * 16;
                while (acc) {
                    const int i = __ffs(acc) - 1;
                    acc &= acc - 1;
                    const int sel = i >> 2, sh = 8 * (i & 3);
                    const uint32_t w0 = sel == 0 ? d.x : sel == 1 ? d.y : sel == 2 ? d.z : d.w;
                    const uint32_t w1 = sel == 0 ? d.y : sel == 1 ? d.z : sel == 2 ? d.w : n0;
                    const uint32_t w2 = sel == 0 ? d.z : sel == 1 ? d.w : sel == 2 ? n0 : n1;
                    const uint32_t lo = __funnelshift_r(w0, w1, sh) & mlo, hi = __funnelshift_r(w1, w2, sh) & mhi;
                    const int64_t g = mc.buf_lo + off + i;
                    if (g < mc.own_lo || g >= mc.own_hi) continue;
                    for (int j = 0; j < p.n_ngrams; j++) {
                        if (grams[j].x != lo || grams[j].y != hi) continue;
                        if (mc.hits_cap) {
                            const unsigned long long ent = ((unsigned long long)g << 8) | (unsigned long long)j;
                            const uint32_t slot = atomicAdd(&scratch[8], 1u);
                            if (slot < 32u) {
                                hbuf[slot] = ent;
                            } else {  // warp buffer full: straight to the list
                                const uint32_t gs = atomicAdd(&mc.counters[CNT_HITS], 1u);
                                if (gs < mc.hits_cap) mc.hits[gs] = ent;
                            }
                        } else {
                            mark_granule(mc.bitmap, mc.glist, mc.glist_cap, mc.counters, (g - mc.buf_lo) >> kGranuleShift);
                            break;
                        }
                    }
                }
            }
            __syncwarp();
            if (mc.hits_cap && scratch[8] >= 16u) {  // warp-uniform (shared memory)
                const uint32_t n = min(scratch[8], 32u);
                uint32_t b0 = 0;
                if (lane == 0) b0 = atomicAdd(&mc.counters[CNT_HITS], n);
                b0 = __shfl_sync(0xFFFFFFFFu, b0, 0);
                if ((uint32_t)lane < n && b0 + lane < mc.hits_cap) mc.hits[b0 + lane] = hbuf[lane];
                __syncwarp();
                if (lane == 0) scratch[8] = 0;
                __syncwarp();
            }
        }
        }
    }
    __syncwarp();
    if (mc.hits_cap && scratch[8]) {
        const uint32_t n = min(scratch[8], 32u);
        uint32_t b0 = 0;
        if (lane == 0) b0 = atomicAdd(&mc.counters[CNT_HITS], n);
        b0 = __shfl_sync(0xFFFFFFFFu, b0, 0);
        if ((uint32_t)lane < n && b0 + lane < mc.hits_cap) mc.hits[b0 + lane] = hbuf[lane];
    }
}

// ------------------------------------------------------------------------------------------------
// Expansion DP -- literal device restatement of levenshtein_ngram.py:8-143 (the CPU test oracle restates
// the same statements independently).  `sub` lives in shared memory, `seq` in global memory; both
// are walked with a stride of +1 (right expansion) or -1 (left expansion, reversed slices of
// levenshtein_ngram.py:186-188).  Returns true and (dist,len), or false for (None, None).
// ------------------------------------------------------------------------------------------------
struct DpScratch {
    uint16_t scores[kMaxPattern + 1];
};

template <int DIR>
__device__ bool expand_short(const uint8_t *sub, int sublen, const uint8_t *seq, int seqlen, int max_l,
                             DpScratch &S, int &dist, int &len) {
    if (sublen == 0) {  // :42-43
        dist = 0;
        len = 0;
        return true;
    }
    for (int j = 0; j < sublen; j++) S.scores[j] = (uint16_t)(j + 1);  // :47
    int min_score = sublen, min_idx = -1;                             // :49-50
    for (int si = 0; si < seqlen; si++) {                             // :52
        const uint8_t ch = seq[DIR * si];
        int a = si, c = si + 1;  // :54-55
        int row_min = 1 << 30;
        for (int j = 0; j < sublen; j++) {  // :56-63
            int b = S.scores[j];
            int v = a + (ch != sub[DIR * j]);
            v = min(v, min(b + 1, c + 1));
            c = v;
            S.scores[j] = (uint16_t)v;
            row_min = min(row_min, v);
            a = b;
        }
        if (c <= min_score) {  // :66-68
            min_score = c;
            min_idx = si;
        } else if (row_min >= min_score) {  // :71-72
            break;
        }
    }
    if (min_score <= max_l) {  // :74
        dist = min_score;
        len = min_idx + 1;
        return true;
    }
    return false;
}

template <int DIR>
__device__ bool expand_long(const uint8_t *sub, int sublen, const uint8_t *seq, int seqlen, int max_l,
                            DpScratch &S, int &dist, int &len) {
    if (sublen == 0) {  // :86-88
        dist = 0;
        len = 0;
        return true;
    }
    for (int j = 0; j < sublen; j++) S.scores[j] = (uint16_t)(j + 1);  // :92
    int min_score = sublen, min_idx = -1;                             // :94-95
    int max_good = max_l;                                             // :96
    int new_start = 0, new_end = sublen - 1;                          // :97-98
    bool ns_none = false;
    for (int si = 0; si < seqlen; si++) {  // :100
        const uint8_t ch = seq[DIR * si];
        const int rstart = new_start;                 // :102
        const int rend = min(sublen, new_end + 1);    // :103
        int a = si, c = si + 1;                       // :105-106
        if (c <= max_good) {                          // :108-113
            new_start = 0;
            ns_none = false;
            new_end = 0;
        } else {
            new_start = 0;
            ns_none = true;
            new_end = -1;
        }
        for (int j = rstart; j < rend; j++) {  // :115-122
            int b = S.scores[j];
            int v = a + (ch != sub[DIR * j]);
            v = min(v, min(b + 1, c + 1));
            c = v;
            S.scores[j] = (uint16_t)v;
            a = b;
            if (c <= max_good) {  // :124-130
                if (ns_none) {
                    ns_none = false;
                    new_start = j;
                }
                new_end = max(new_end, j + 1 + (max_good - c));
            }
        }
        if (ns_none) break;                     // :133-134
        if (rend == sublen && c <= min_score) {  // :137-141
            min_score = c;
            min_idx = si;
            if (min_score < max_good) max_good = min_score;
        }
    }
    if (min_score <= max_l) {  // :143
        dist = min_score;
        len = min_idx + 1;
        return true;
    }
    return false;
}

// Register-resident variant for sub-sequences of at most kRegSub characters (the common case: the
// expansions of a 20-byte pattern are 2..14 characters long): same statements as above, but the DP
// row lives in registers (fully unrolled, predicated) instead of local memory.
constexpr int kRegSub = 16;

// One routine for both reference variants (levenshtein_ngram.py:22-74 and :77-143) when the row fits
// the registers: the variant is a per-lane FLAG, not a different function, so the lanes of a warp that
// expand different hits (different lengths, different variants) stay converged and the warp pays for
// the longest expansion instead of the sum of all of them.
template <int DIR>
__device__ bool expand_uni_reg(const uint8_t *sub, int sublen, const uint8_t *seq, int seqlen, int max_l, int &dist,
                               int &len) {
    if (sublen == 0) {
        dist = 0;
        len = 0;
        return true;
    }
    const bool is_long = sublen > max(2 * max_l, 10);  // levenshtein_ngram.py:16
    int sc[kRegSub];
    uint8_t pc[kRegSub];
#pragma unroll
    for (int j = 0; j < kRegSub; j++) {
        sc[j] = j + 1;
        pc[j] = j < sublen ? sub[DIR * j] : 0;
    }
    int min_score = sublen, min_idx = -1;
    int max_good = max_l;
    int new_start = 0, new_end = sublen - 1;
    bool ns_none = false;
    for (int si = 0; si < seqlen; si++) {
        const uint8_t ch = seq[DIR * si];
        const int rstart = is_long ? new_start : 0;
        const int rend = is_long ? min(sublen, new_end + 1) : sublen;
        int a = si, c = si + 1;
        if (is_long) {
            new_start = 0;
            ns_none = !(c <= max_good);
            new_end = ns_none ? -1 : 0;
        }
        int row_min = 1 << 30;
#pragma unroll
        for (int j = 0; j < kRegSub; j++) {
            if (j >= rstart && j < rend) {
                const int b = sc[j];
                int v = a + (ch != pc[j]);
                v = min(v, min(b + 1, c + 1));
                c = v;
                sc[j] = v;
                row_min = min(row_min, v);
                a = b;
                if (is_long && c <= max_good) {
                    if (ns_none) {
                        ns_none = false;
                        new_start = j;
                    }
                    new_end = max(new_end, j + 1 + (max_good - c));
                }
            }
        }
        if (is_long) {
            if (ns_none) break;
            if (rend == sublen && c <= min_score) {
                min_score = c;
                min_idx = si;
                if (min_score < max_good) max_good = min_score;
            }
        } else {
            if (c <= min_score) {
                min_score = c;
                min_idx = si;
            } else if (row_min >= min_score) {
                break;
            }
        }
    }
    if (min_score <= max_l) {
        dist = min_score;
        len = min_idx + 1;
        return true;
    }
    return false;
}

template <int DIR>
__device__ __forceinline__ bool expand_any(const uint8_t *sub, int sublen, const uint8_t *seq,
                                           int seqlen, int max_l, DpScratch &S, int &dist, int &len) {
    if (sublen <= kRegSub) return expand_uni_reg<DIR>(sub, sublen, seq, seqlen, max_l, dist, len);
    if (sublen > max(2 * max_l, 10))  // levenshtein_ngram.py:16
        return expand_long<DIR>(sub, sublen, seq, seqlen, max_l, S, dist, len);
    return expand_short<DIR>(sub, sublen, seq, seqlen, max_l, S, dist, len);
}

// ------------------------------------------------------------------------------------------------
// Bit-parallel expansion (patterns of at most 64 bytes): the same function _expand computes
// (levenshtein_ngram.py:8-143), evaluated with the Myers / Hyyro bit-vector recurrence instead of the
// reference's cell-by-cell lists.  One machine word holds the vertical deltas of one DP row of the
// reference (= one haystack character); D[len(sub)][l] is tracked from the horizontal delta at the last
// pattern position, with +1 shifted in at position 0 because D[0][l] = l (prefix-anchored distance).
//   * "long" variant (_py_expand_long, :77-143): the exact rule -- minimise over prefix lengths l, ties to
//     the largest l.  Its Ukkonen band only prunes cells that cannot matter (SURVEY a5), so the full
//     recurrence returns the same (dist, len).
//   * "short" variant (_py_expand_short, :22-74): same scan plus the reference's early break
//     `elif min(row) >= min_score: break` (:71-72, SURVEY F6); the row minimum is recovered from the
//     vertical deltas (a running sum over the <= max(2k,10) positions), only on rows that do not improve.
// Both were checked against the oracle on 600 000 random cases on the CPU before being written here;
// tests/test_gpu_oracle.py / test_gpu_expand.py pin the device code.
// The Eq masks come from ONE table per pattern, PM[c] = {i : P[i] == c}: the right sub-pattern
// P[s+L:] is PM >> (s+L); the left one, reversed P[:s], is the bit reversal of PM shifted down.
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ void build_pm(unsigned long long *sPM, const uint8_t *P, int m, int tid, int nthreads) {
    for (int c = tid; c < 256; c += nthreads) {
        unsigned long long v = 0;
        for (int i = 0; i < m && i < 64; i++) v |= (unsigned long long)(P[i] == c) << i;
        sPM[c] = v;
    }
}

template <typename Wt, int DIR>
__device__ __forceinline__ bool expand_bp(const unsigned long long *sPM, int s_off, int sublen, const uint8_t *seq,
                                          int seqlen, int max_l, int &dist, int &len, int variant = 0) {
    // DIR = +1: sub = P[s_off : s_off+sublen];  DIR = -1: sub = reversed P[:s_off] (sublen == s_off)
    if (sublen == 0) {  // :42-43, :86-88
        dist = 0;
        len = 0;
        return true;
    }
    // levenshtein_ngram.py:16 (variant 1 / 2 force _py_expand_short / _py_expand_long: fzb_debug_expand only)
    const bool is_long = variant == 0 ? sublen > max(2 * max_l, 10) : variant == 2;
    Wt VP = ~(Wt)0, VN = 0;
    const Wt top = (Wt)1 << (sublen - 1);
    int score = sublen, min_score = sublen, min_idx = -1;  // :49-50, :94-95
    for (int si = 0; si < seqlen; si++) {
        const unsigned long long pm = sPM[seq[DIR * si]];
        const Wt Eq = DIR > 0 ? (Wt)(pm >> s_off) : (Wt)(__brevll(pm) >> (64 - s_off));
        const Wt Xv = Eq | VN;
        const Wt Xh = (((Eq & VP) + VP) ^ VP) | Eq;
        Wt HP = VN | ~(Xh | VP);
        Wt HN = VP & Xh;
        score += (HP & top) ? 1 : 0;
        score -= (HN & top) ? 1 : 0;
        HP = (HP << 1) | (Wt)1;  // D[0][l] = l: the top row steps by +1
        HN <<= 1;
        VP = HN | ~(Xv | HP);
        VN = HP & Xv;
        if (score <= min_score) {  // :66-68, :137-139 (ties -> the later row)
            min_score = score;
            min_idx = si;
        } else if (!is_long) {  // :71-72: stop if no cell of this row is below the best so far
            int v = si + 1, row_min = 1 << 30;
            for (int j = 0; j < sublen; j++) {
                v += (int)((VP >> j) & 1) - (int)((VN >> j) & 1);
                row_min = min(row_min, v);
            }
            if (row_min >= min_score) break;
        }
    }
    if (min_score <= max_l) {  // :74, :143
        dist = min_score;
        len = min_idx + 1;
        return true;
    }
    return false;
}

// The cell-by-cell routines need a DP row in local memory; the bit-parallel modes must not carry it.
template <int VM>
struct DpHolder {
    __device__ __forceinline__ DpScratch *get() { return nullptr; }
};
template <>
struct DpHolder<2> {
    DpScratch s;
    __device__ __forceinline__ DpScratch *get() { return &s; }
};

// Same recurrence with the Eq mask computed on the fly from the sub-pattern's characters (no per-pattern table):
// used where every LANE verifies a different pattern (k_verify_mhits, batch_kernels.cuh) and a 2 KiB table per lane
// is out of the question.  sub[DIR * i] is character i of the sub-pattern; sublen <= 32.
template <int DIR>
__device__ __forceinline__ bool expand_bp_otf(const uint8_t *sub, int sublen, const uint8_t *seq, int seqlen,
                                              int max_l, int &dist, int &len) {
    if (sublen == 0) {
        dist = 0;
        len = 0;
        return true;
    }
    const bool is_long = sublen > max(2 * max_l, 10);  // levenshtein_ngram.py:16
    uint32_t VP = ~0u, VN = 0;
    const uint32_t top = 1u << (sublen - 1);
    int score = sublen, min_score = sublen, min_idx = -1;
    for (int si = 0; si < seqlen; si++) {
        const uint8_t ch = seq[DIR * si];
        uint32_t Eq = 0;
        for (int i = 0; i < sublen; i++) Eq |= (uint32_t)(sub[DIR * i] == ch) << i;
        const uint32_t Xv = Eq | VN;
        const uint32_t Xh = (((Eq & VP) + VP) ^ VP) | Eq;
        uint32_t HP = VN | ~(Xh | VP);
        uint32_t HN = VP & Xh;
        score += (HP & top) ? 1 : 0;
        score -= (HN & top) ? 1 : 0;
        HP = (HP << 1) | 1u;
        HN <<= 1;
        VP = HN | ~(Xv | HP);
        VN = HP & Xv;
        if (score <= min_score) {
            min_score = score;
            min_idx = si;
        } else if (!is_long) {
            int v = si + 1, row_min = 1 << 30;
            for (int j = 0; j < sublen; j++) {
                v += (int)((VP >> j) & 1) - (int)((VN >> j) & 1);
                row_min = min(row_min, v);
            }
            if (row_min >= min_score) break;
        }
    }
    if (min_score <= max_l) {
        dist = min_score;
        len = min_idx + 1;
        return true;
    }
    return false;
}

// Verification mode of a pattern: 0 = bit-parallel, 32-bit words (m <= 64, m-L <= 32); 1 = bit-parallel, 64-bit
// words (m <= 64); 2 = cell-by-cell DP with the row in registers / local memory (longer patterns).
__host__ __device__ __forceinline__ int verify_mode(int m, int L) { return m > 64 ? 2 : (m - L <= 32 ? 0 : 1); }

// ------------------------------------------------------------------------------------------------
// Verify kernel for the Levenshtein n-gram route (levenshtein_ngram.py:159-198).  One warp per
// marked granule; lane <-> anchor position.  Boundary rules are evaluated in GLOBAL coordinates
// (0 and N), never at shard seams.
// ------------------------------------------------------------------------------------------------
constexpr int kVerifyThreads = 128;

// canonical order (start, end, dist): start < 2^46, end-start < 2^10, dist < 2^8
__device__ __forceinline__ uint64_t canonical_key(const RawRec &r) {
    return ((uint64_t)r.start << 18) | ((uint64_t)(r.end - r.start) << 8) | (uint64_t)r.dist;
}

// Appends one raw match.  The packed canonical keys k_post orders and consolidates live in a parallel array
// right behind the records, with their own counter: a caller that KNOWS another lane of its warp is emitting
// the identical (start, end, dist) right now passes with_key = false for all but one of them -- duplicates
// change neither the groups nor the winners of consolidate_overlapping_matches, and the n-gram search finds
// most occurrences once per n-gram (levenshtein_ngram.py:194-198 yields them all; the raw stream keeps them).
__device__ __forceinline__ void emit(RawRec *out, uint32_t cap, uint32_t *counters, int64_t start,
                                     int64_t end, int64_t idx, int dist, int ngram, bool with_key = true) {
    uint32_t slot = atomicAdd(&counters[CNT_OUT], 1u);
    RawRec r;
    r.start = start;
    r.end = end;
    r.idx = idx;
    r.dist = dist;
    r.ngram = ngram;
    if (slot < cap) out[slot] = r;
    if (with_key) {
        slot = atomicAdd(&counters[CNT_KEYS], 1u);
        if (slot < cap) reinterpret_cast<uint64_t *>(out + cap)[slot] = canonical_key(r);
    }
}

// Window staging: a marked granule [gbase, gbase+64) only ever needs H[gbase-(m+k) : gbase+64+m+k)
// (every anchor's n-gram test and both expansions stay inside it), so the warp copies that window
// into shared memory with ONE round trip to DRAM and all further reads are shared-memory reads --
// the compares and the DP are chains of dependent byte reads, which would otherwise each pay the
// full DRAM latency (the scan streamed the haystack past the caches).
constexpr int kWinBytes = 64 + 2 * (2 * kMaxPattern) + 32;  // 1116
constexpr int kWinWords = (kWinBytes + 3) / 4;

// Loads the window of granule `gbase` into sWin; returns the global position of sWin[0].
template <class PT>
__device__ __forceinline__ int64_t stage_window(const PT &p, int64_t gbase, int halo, int lane,
                                                uint32_t *sWin) {
    int64_t wlo = max(gbase - halo, p.buf_lo);
    int64_t whi = min(gbase + kGranule + halo, p.buf_lo + p.buf_len);
    const int64_t alo = wlo & ~(int64_t)3;  // buf_lo is a multiple of 16, so global and buffer alignment agree
    const int nwords = (int)((whi - alo + 3) >> 2);
    const uint32_t *src = reinterpret_cast<const uint32_t *>(p.H + (alo - p.buf_lo));
    __syncwarp();
    for (int w = lane; w < nwords; w += 32) sWin[w] = __ldg(src + w);  // padded buffer: reads past whi are safe
    __syncwarp();
    return alo;
}

// All lanes of the warp call this together (lanes without an anchor pass valid = false).  Each lane
// first finds the next n-gram that really occurs at its anchor (cheap), THEN the lanes that found one
// run the two expansions side by side (converged), and the search for further n-grams resumes.
// VM = verify_mode(m, L); S is only used (and only non-null) in mode 2.  Mode 3 (batch hit lists): m, k, L, the pattern
// bytes sP and the tag differ from lane to lane.
// PT: ScanParams, or the per-work-item VerifyCtx of the multi-pattern kernels (batch_kernels.cuh); `tag` is OR-ed
// into the n-gram field of the emitted records (pattern number << 8 in a batch).
struct VerifyCtx {
    const uint8_t *H;
    int64_t buf_lo, buf_len, N, own_lo, own_hi;
    int32_t m, k, L, n_ngrams;
};

template <int VM, class PT>
__device__ void verify_anchor_lev(const PT &p, const uint8_t *sP, const unsigned long long *sPM,
                                  const uint8_t *W, int64_t idx, bool valid, DpScratch *S, RawRec *out, uint32_t cap,
                                  uint32_t *counters, int j_lo, int j_hi, int tag = 0) {
    // W[g] is the haystack byte at global position g (shared-memory window); n-grams j_lo..j_hi-1
    const int m = p.m, k = p.k, L = p.L;
    const int64_t N = p.N;
    const uint8_t *h = W + idx;
    int j = valid ? j_lo : j_hi;
    for (;;) {
        for (; j < j_hi; j++) {  // next n-gram hit at this anchor
            const int s = j * L;  // :170
            // search window of n-gram j, clamped like search_exact.py:29-30   (:174-176)
            int64_t ws = max((int64_t)0, (int64_t)(s - k));
            int64_t we = min(N, N - m + s + L + k);
            ws = max((int64_t)0, min(ws, N));
            we = max(ws, min(we, N));
            if (idx < ws || idx + L > we) continue;
            bool eq = true;
            for (int i = 0; i < L; i++) {
                if (h[i] != sP[s + i]) {
                    eq = false;
                    break;
                }
            }
            if (eq) break;
        }
        const bool have = j < j_hi;
        if (!__any_sync(0xFFFFFFFFu, have)) return;
        const int s = have ? j * L : 0;
        const int64_t p0 = idx - s;
        // right: _expand(P[s+L:], H[idx+L : p0+m+k], k)   (:178-182)
        int dr = 0, rs = 0, dl = 0, ls = 0;
        bool ok = have;
        if (ok) {
            const int64_t rhi = min(N, p0 + m + k);
            const int rlen = (int)max((int64_t)0, rhi - (idx + L));
            if (VM == 3)  // per-lane patterns: Eq on the fly (m - L <= 32)
                ok = expand_bp_otf<1>(sP + s + L, m - s - L, h + L, rlen, k, dr, rs);
            else if (VM == 0)
                ok = expand_bp<uint32_t, 1>(sPM, s + L, m - s - L, h + L, rlen, k, dr, rs);
            else if (VM == 1)
                ok = expand_bp<unsigned long long, 1>(sPM, s + L, m - s - L, h + L, rlen, k, dr, rs);
            else
                ok = expand_any<1>(sP + s + L, m - s - L, h + L, rlen, k, *S, dr, rs);
        }
        // left: _expand(P[:s][::-1], H[max(0,p0-(k-dr)) : idx][::-1], k-dr)   (:185-189)
        if (ok) {
            const int64_t llo = max((int64_t)0, p0 - (k - dr));
            const int llen = (int)max((int64_t)0, idx - llo);
            if (VM == 3)
                ok = expand_bp_otf<-1>(sP + s - 1, s, h - 1, llen, k - dr, dl, ls);
            else if (VM == 0)
                ok = expand_bp<uint32_t, -1>(sPM, s, s, h - 1, llen, k - dr, dl, ls);
            else if (VM == 1)
                ok = expand_bp<unsigned long long, -1>(sPM, s, s, h - 1, llen, k - dr, dl, ls);
            else
                ok = expand_any<-1>(sP + s - 1, s, h - 1, llen, k - dr, *S, dl, ls);
        }
        // :194-198.  Lanes of this warp that found the SAME match through different n-grams share one key.
        const unsigned okm = __ballot_sync(0xFFFFFFFFu, ok);
        if (ok) {
            const unsigned long long ident = ((unsigned long long)(idx - ls) << 18) |
                                             ((unsigned long long)(L + rs + ls) << 8) | (unsigned long long)(dl + dr);
            const unsigned peers = __match_any_sync(okm, ident);
            emit(out, cap, counters, idx - ls, idx + L + rs, idx, dl + dr, j | tag,
                 (__ffs(peers) - 1) == (int)(threadIdx.x & 31));
        }
        j++;
    }
}

// Work distribution.  The filters append every newly marked granule to a work list (mark_granule) and
// the verify kernel hands ONE GRANULE TO ONE WARP through an atomic work counter, so clustered matches (the realistic case) spread over the
// whole GPU instead of serialising on the warp that owns their bitmap words.  Each processed granule
// clears its own bit; if the list overflows (dense candidates, e.g. small alphabets) the bits left
// set are swept by the bitmap-scanning fallback loop of the same kernel launched in "scan" mode.
template <int VM, class PT>
__device__ __forceinline__ void verify_granule_lev(const PT &p, const uint8_t *sP,
                                                   const unsigned long long *sPM, uint32_t *sWin, int64_t granule,
                                                   int lane, DpScratch *S, RawRec *out, uint32_t cap,
                                                   uint32_t *counters, int tag = 0) {
    const int64_t gbase = p.buf_lo + (granule << kGranuleShift);
    const int64_t alo = stage_window(p, gbase, p.m + p.k, lane, sWin);
    const uint8_t *W = reinterpret_cast<const uint8_t *>(sWin) - alo;
#pragma unroll 1
    for (int half = 0; half < kGranule / 32; half++) {
        const int64_t idx = gbase + half * 32 + lane;
        verify_anchor_lev<VM>(p, sP, sPM, W, idx, idx >= p.own_lo && idx < p.own_hi, S, out, cap, counters, 0,
                              p.n_ngrams, tag);
    }
}

// scan_mode == 0: process glist[0 .. CNT_GRAN) one granule per warp (the normal case: ONE verify launch per search).
// scan_mode == 1: no list -- sweep the whole bitmap (the host's second attempt after the list overflowed).
template <int VM>
__global__ void __launch_bounds__(kVerifyThreads)
k_verify_lev(const ScanParams p, uint64_t bitmap_words, const uint32_t *glist, uint32_t glist_cap, int scan_mode,
             RawRec *out, uint32_t cap, uint32_t *counters) {
    __shared__ uint8_t sP[256];
    __shared__ unsigned long long sPM[VM < 2 ? 256 : 1];
    __shared__ uint32_t sWinAll[kVerifyThreads / 32][kWinWords];
    const uint32_t ngran = counters[CNT_GRAN];
    for (int i = threadIdx.x; i < 256; i += blockDim.x) sP[i] = p.P[i];
    if (VM < 2) build_pm(sPM, p.P, p.m, threadIdx.x, blockDim.x);
    __syncthreads();
    DpHolder<VM> dp_holder;
    DpScratch *S = dp_holder.get();
    const int lane = threadIdx.x & 31;
    uint32_t *sWin = sWinAll[threadIdx.x >> 5];
    if (!scan_mode) {
        if (ngran > glist_cap) {  // the work list overflowed (pathologically dense marks): the host repeats the search in
            if (blockIdx.x == 0 && threadIdx.x == 0) counters[CNT_OVERFLOW] = 1;  // bitmap mode (scan_mode = 1, no list)
            return;
        }
        const uint32_t nitems = ngran;
        for (;;) {
            uint32_t item = 0;
            if (lane == 0) item = atomicAdd(&counters[CNT_WORK], 1u);
            item = __shfl_sync(0xFFFFFFFFu, item, 0);
            if (item >= nitems) break;
            const uint32_t g = glist[item];
            verify_granule_lev<VM>(p, sP, sPM, sWin, (int64_t)g, lane, S, out, cap, counters);
            if (lane == 0) atomicAnd(&p.bitmap[g >> 5], ~(1u << (g & 31)));
        }
        if (blockIdx.x == 0 && threadIdx.x == 0) atomicAdd(&counters[CNT_CAND], nitems);
        return;
    }
    const uint64_t gwarp = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const uint64_t nwarps = ((uint64_t)gridDim.x * blockDim.x) >> 5;
    for (uint64_t wbase = gwarp * 32; wbase < bitmap_words; wbase += nwarps * 32) {
        const uint64_t wi = wbase + lane;
        uint32_t bits = wi < bitmap_words ? p.bitmap[wi] : 0u;
        if (bits) p.bitmap[wi] = 0u;  // consumed: the bitmap is all-zero again when the kernel ends
        unsigned active = __ballot_sync(0xFFFFFFFFu, bits != 0);
        while (active) {
            const int src = __ffs(active) - 1;
            active &= active - 1;
            uint32_t b = __shfl_sync(0xFFFFFFFFu, bits, src);
            if (lane == 0) atomicAdd(&counters[CNT_CAND], (uint32_t)__popc(b));
            while (b) {
                const int bit = __ffs(b) - 1;
                b &= b - 1;
                verify_granule_lev<VM>(p, sP, sPM, sWin, (int64_t)(wbase + src) * 32 + bit, lane, S, out, cap,
                                       counters);
            }
        }
    }
}

// ------------------------------------------------------------------------------------------------
// Hit-list verification (dense route on low-entropy data, where hits are many): ONE LANE PER HIT.
// Each lane copies the window of its own hit, H[p0-k : p0+m+k), into its private slot of shared
// memory (one round trip, independent loads), then runs the n-gram compare and both expansions from
// there -- 32 hits verified in parallel per warp instead of one hit per granule per warp.
// ------------------------------------------------------------------------------------------------
constexpr int kHitSlotBytes = 144;  // per-lane window slot: m + 2k + alignment slack must fit
constexpr int kHitThreads = 128;

template <int VM>
__global__ void __launch_bounds__(kHitThreads)
k_verify_hits(const ScanParams p, RawRec *out, uint32_t cap, uint32_t *counters) {
    __shared__ uint8_t sP[256];
    __shared__ unsigned long long sPM[VM < 2 ? 256 : 1];
    __shared__ __align__(16) uint8_t slots[kHitThreads][kHitSlotBytes];
    for (int i = threadIdx.x; i < 256; i += blockDim.x) sP[i] = p.P[i];
    if (VM < 2) build_pm(sPM, p.P, p.m, threadIdx.x, blockDim.x);
    __syncthreads();
    const uint32_t nhits = counters[CNT_HITS];
    if (nhits > p.hits_cap) {  // list overflowed: the host repeats the search in granule mode
        if (blockIdx.x == 0 && threadIdx.x == 0) counters[CNT_OVERFLOW] = 1;
        return;
    }
    DpHolder<VM> dp_holder;
    DpScratch *S = dp_holder.get();
    const int lane = threadIdx.x & 31;
    uint8_t *slot = slots[threadIdx.x];
    for (;;) {
        uint32_t base = 0;
        if (lane == 0) base = atomicAdd(&counters[CNT_HITWORK], 32u);
        base = __shfl_sync(0xFFFFFFFFu, base, 0);
        if (base >= nhits) break;
        const uint32_t item = base + lane;
        const bool valid = item < nhits;
        int64_t idx = 0, alo = 0;
        int j = 0;
        if (valid) {
            const uint64_t hv = p.hits[item];
            idx = (int64_t)(hv >> 8);
            j = (int)(hv & 0xFFu);
            const int64_t p0 = idx - (int64_t)j * p.L;
            const int64_t wlo = max(max(p0 - p.k, (int64_t)0), p.buf_lo);
            const int64_t whi = min(min(p0 + p.m + p.k, p.N), p.buf_lo + p.buf_len);
            alo = wlo & ~(int64_t)3;
            const int nwords = (int)((whi - alo + 3) >> 2);
            const uint32_t *src = reinterpret_cast<const uint32_t *>(p.H + (alo - p.buf_lo));
            uint32_t *dst = reinterpret_cast<uint32_t *>(slot);
            for (int w = 0; w < nwords; w++) dst[w] = __ldg(src + w);
        }
        verify_anchor_lev<VM>(p, sP, sPM, slot - alo, idx, valid, S, out, cap, counters, j, j + 1);  // whole warp
    }
    if (blockIdx.x == 0 && threadIdx.x == 0) atomicAdd(&counters[CNT_CAND], nhits);
}

// ------------------------------------------------------------------------------------------------
// Synthetic corpus fill (bench / tests): byte i = alphabet[hash(seed, i)], counter based.
// ------------------------------------------------------------------------------------------------
__global__ void k_fill_synth(uint8_t *H, int64_t buf_lo, int64_t nwords, uint64_t seed,
                             const uint8_t *alphabet_g, uint32_t alen) {
    __shared__ uint8_t alphabet[256];
    for (int i = threadIdx.x; i < (int)alen; i += blockDim.x) alphabet[i] = alphabet_g[i];
    __syncthreads();
    uint32_t *W = reinterpret_cast<uint32_t *>(H);
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    // buf_lo is required to be a multiple of 4 by the host
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < nwords; i += stride)
        W[i] = synth_word(seed, (uint64_t)(buf_lo / 4 + i), alphabet, alen);
}

}  // namespace fzb
