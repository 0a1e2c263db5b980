// batch_kernels.cuh -- many patterns over one haystack in ONE pass (BASELINE.json configs[4]).
//
// The reference has no batch API: a caller loops find_near_matches over the patterns
// (src/fuzzysearch/__init__.py:35-57), reading the haystack (k+1) times per pattern.  Here every pattern for
// which the q-sample lemma of k_filter_sampled holds (floor((m-k-3)/4) >= k+1, m <= 64) shares one scan:
//   k_filter_multi  streams the haystack once.  The 4-grams of ALL those patterns (~30 K for 800 patterns) set bits
//        in a 2^20-bit table in shared memory (128 KiB, one CTA of 1024 threads per SM); each 4-byte-aligned
//        haystack word costs one hash + one bit test.  Table hits (~3 %: a Bloom filter at 3 % load) are confirmed by
//        the flagged lane itself against an L2-resident open-addressing table gram -> postings (pattern, offset);
//        a real hit of pattern p at offset o marks the granules that can hold an n-gram anchor of an occurrence
//        containing that word, anchors [g-o-k, g-o+k+m-L] (the word is aligned with pattern offset o up to k
//        insertions/deletions).  (pattern, granule) pairs are de-duplicated by a device hash set (CAS insert)
//        and the inserting thread appends the pair to the work list.
//   k_verify_multi  one warp per (pattern, granule): loads that pattern, builds its bit-parallel match table
//        in shared memory and runs the same verify_granule_lev as the single-pattern search; records are tagged
//        with the pattern number.  The set slot is cleared on the way out (the set is empty between batches).
// The host splits the records by pattern and consolidates each list (api.cu).
#pragma once
#include "lp_kernels.cuh"

namespace fzb {

constexpr int kMultiThreads = 1024;
constexpr int kMultiTblBits = 20;
constexpr int kMultiTblWords = 1 << (kMultiTblBits - 5);  // 32768 words = 128 KiB
constexpr size_t kMultiSmem = (size_t)kMultiTblWords * 4;
constexpr int kMultiUnroll = 4;                            // uint4 loads in flight per thread
constexpr int kMultiTileVecs = kMultiThreads * kMultiUnroll;
constexpr uint32_t kGramMul = 0x85EBCA77u;
constexpr int kMulti2Bits = 23;                            // 1 MiB second-level bit table
constexpr int kMulti2Words = 1 << (kMulti2Bits - 5);
constexpr uint32_t kGramMul2 = 0xC2B2AE35u;
__host__ __device__ __forceinline__ uint32_t multi_hash2(uint32_t w) { return ((w ^ (w >> 15)) * kGramMul2) >> (32 - kMulti2Bits); }
constexpr int kBatchMaxM = 64;

struct BatchPat {  // device copy of one pattern
    uint8_t P[kBatchMaxM];
    int32_t m, k, L, n_ngrams;
};

struct WorkItem {
    uint32_t pid, granule, slot, pad;
};

struct MultiParams {
    const uint8_t *H;
    int64_t buf_lo, buf_len, N, own_lo, own_hi;
    const uint32_t *bits;      // global copy of the bit table (kMultiTblWords words)
    const uint32_t *bits2;     // second-level table (kMulti2Words words, L2-resident, independent hash): a word that
                               // passes the shared-memory test (3 % false positives) must pass this one too before a
                               // lane walks the postings (k_filter_multi only; nullptr = skip)
    const uint2 *gtab;         // open addressing: .x gram, .y = first posting | count << 24 (0 = empty slot)
    uint32_t gtab_mask;
    const uint32_t *postings;  // pid << 8 | offset
    const uint32_t *pinfo;     // per pattern: m | k << 8 | L << 16
    unsigned long long *set;   // de-duplication set of (pid << 32 | granule) + 1, 0 = empty
    uint32_t set_mask;
    WorkItem *work;
    uint32_t work_cap;
    uint32_t *counters;        // CNT_GRAN = work items appended, CNT_OVERFLOW
};

__device__ __forceinline__ uint32_t multi_hash(uint32_t w) { return (w * kHashMul) >> (32 - kMultiTblBits); }

// one (pattern, granule) pair: insert into the set; the inserter appends the work item
__device__ __forceinline__ void multi_mark(const MultiParams &p, uint32_t pid, uint32_t granule) {
    const unsigned long long key = (((unsigned long long)pid << 32) | granule) + 1ull;
    uint32_t slot = (uint32_t)((key * 0x9E3779B97F4A7C15ull) >> 32) & p.set_mask;
    for (uint32_t probe = 0; probe < 256; probe++) {
        const unsigned long long old = atomicCAS(&p.set[slot], 0ull, key);
        if (old == key) return;  // somebody marked it already
        if (old == 0ull) {
            const uint32_t w = atomicAdd(&p.counters[CNT_GRAN], 1u);
            if (w < p.work_cap) {
                WorkItem it;
                it.pid = pid;
                it.granule = granule;
                it.slot = slot;
                it.pad = 0;
                p.work[w] = it;
            } else {
                atomicExch(&p.counters[CNT_OVERFLOW], 1u);
            }
            return;
        }
        slot = (slot + 1) & p.set_mask;
    }
    atomicExch(&p.counters[CNT_OVERFLOW], 1u);  // set too full: the host redoes the batch pattern by pattern
}

// a haystack word whose table bit is set: look the gram up, mark the granules of every pattern that has it
__device__ __noinline__ void multi_confirm(const MultiParams &p, uint32_t w, int64_t word_off) {
    uint32_t slot = (w * kGramMul) & p.gtab_mask;
    for (;;) {
        const uint2 e = __ldg(p.gtab + slot);
        if (e.y == 0u) return;  // not a pattern gram: a false positive of the bit table
        if (e.x == w) {
            const uint32_t first = e.y & 0xFFFFFFu, cnt = e.y >> 24;
            const int64_t g = p.buf_lo + word_off;
            for (uint32_t i = 0; i < cnt; i++) {
                const uint32_t post = __ldg(p.postings + first + i);
                const uint32_t pid = post >> 8;
                const int o = (int)(post & 0xFFu);
                const uint32_t info = __ldg(p.pinfo + pid);
                const int m = (int)(info & 0xFFu), k = (int)((info >> 8) & 0xFFu), L = (int)((info >> 16) & 0xFFu);
                int64_t lo = g - o - k, hi = g - o + k + (m - L);  // anchors of occurrences aligning this word with offset o
                if (lo < p.own_lo) lo = p.own_lo;
                if (hi > p.own_hi - 1) hi = p.own_hi - 1;
                if (lo > hi) continue;
                const int64_t g0 = (lo - p.buf_lo) >> kGranuleShift, g1 = (hi - p.buf_lo) >> kGranuleShift;
                for (int64_t gr = g0; gr <= g1; gr++) multi_mark(p, pid, (uint32_t)gr);
            }
            // keep probing: a gram with more than 255 postings occupies several slots
        }
        slot = (slot + 1) & p.gtab_mask;
    }
}

__global__ void __launch_bounds__(kMultiThreads, 1)
k_filter_multi(const __grid_constant__ MultiParams p, int64_t nvec, int64_t ntiles) {
    extern __shared__ __align__(16) uint32_t mtbl[];
    for (int i = threadIdx.x; i < kMultiTblWords / 4; i += kMultiThreads)
        reinterpret_cast<uint4 *>(mtbl)[i] = __ldg(reinterpret_cast<const uint4 *>(p.bits) + i);
    __syncthreads();
    const uint4 *base = reinterpret_cast<const uint4 *>(p.H);
    for (int64_t t = blockIdx.x; t < ntiles; t += gridDim.x) {
        const int64_t v0 = t * kMultiTileVecs + threadIdx.x;
        uint4 d[kMultiUnroll];
#pragma unroll
        for (int u = 0; u < kMultiUnroll; u++) {
            const int64_t v = v0 + (int64_t)u * kMultiThreads;
            d[u] = (v < nvec) ? ldg_stream(base + v) : make_uint4(0, 0, 0, 0);
        }
        uint32_t acc = 0;  // bit (15 - 4u - i) <-> word i of load u
#pragma unroll
        for (int u = 0; u < kMultiUnroll; u++) {
            const uint32_t ws[4] = {d[u].x, d[u].y, d[u].z, d[u].w};
#pragma unroll
            for (int i = 0; i < 4; i++) {
                const uint32_t h = multi_hash(ws[i]);
                acc = acc * 2u + ((mtbl[h >> 5] >> (h & 31u)) & 1u);
            }
        }
        if (acc) {  // ~3 % of the words: the flagged lane confirms its own words (independent L2 probes)
#pragma unroll
            for (int u = 0; u < kMultiUnroll; u++) {
                const uint32_t nib = (acc >> (4 * (kMultiUnroll - 1 - u))) & 0xFu;
                if (!nib) continue;
                const int64_t off = (v0 + (int64_t)u * kMultiThreads) * 16;
                if (off >= p.buf_len) continue;  // zero padding behind the buffer
                const uint32_t ws[4] = {d[u].x, d[u].y, d[u].z, d[u].w};
#pragma unroll
                for (int i = 0; i < 4; i++) {
                    if (!(nib & (8u >> i))) continue;
                    const uint32_t h2 = multi_hash2(ws[i]);
                    if (p.bits2 && !((__ldg(p.bits2 + (h2 >> 5)) >> (h2 & 31u)) & 1u)) continue;  // second level: L2
                    multi_confirm(p, ws[i], off + 4 * i);
                }
            }
        }
    }
}

// ------------------------------------------------------------------------------------------------
// The patterns the q-sample lemma does NOT cover (short patterns / large k: "dense" class) share a scan too, built on
// the reference's own filter -- at least one of the n-grams P[jL:(j+1)L] occurs exactly (levenshtein_ngram.py:159-198):
//   k_filter_mdense  tests the 3-byte prefix of every n-gram of every such pattern (every n-gram is >= 3 bytes on the
//        n-gram route) at EVERY haystack position against the same kind of 2^20-bit table (funnel shift, one hash,
//        one bit test per position); a flagged lane probes the prefix -> postings (pattern, n-gram) table, compares
//        the rest of the n-gram with the text and appends a HIT (pattern, n-gram, position) -- buffered per CTA in
//        shared memory, one global atomic per flush.
//   k_verify_mhits   one hit per LANE (like k_verify_hits): the lane stages its window and its own pattern in
//        private shared-memory slots and runs verify_anchor_lev for that one n-gram, computing the Eq masks of the
//        bit-parallel expansion on the fly (every lane has a different pattern).
// ------------------------------------------------------------------------------------------------
constexpr int kMdBuf = 3072;     // hits buffered per CTA
constexpr int kMdFlush = 1024;
constexpr size_t kMdenseSmem = kMultiSmem + (size_t)kMdBuf * 8 + 16;
enum { CNT_MHITS = 7, CNT_MHITWORK = 8 };

struct MdenseParams {
    MultiParams mp;             // table pointers as for k_filter_multi (gtab keyed by the 3-byte prefix, postings pid << 8 | j)
    const BatchPat *pats;
    unsigned long long *hits;   // (idx - buf_lo) | j << 40 | pid << 48: buffer-relative, so buf_len < 2^40 (check_shard)
    uint32_t hits_cap;
};

// -> true when this append brought the CTA buffer to its flush threshold
__device__ __forceinline__ bool mdense_append(const MdenseParams &p, unsigned long long *sBuf, uint32_t *sN,
                                              unsigned long long hit) {
    const uint32_t slot = atomicAdd(sN, 1u);
    if (slot < (uint32_t)kMdBuf) {
        sBuf[slot] = hit;
    } else {  // CTA buffer full (a very dense tile): straight to the global list
        const uint32_t g = atomicAdd(&p.mp.counters[CNT_MHITS], 1u);
        if (g < p.hits_cap) p.hits[g] = hit;
    }
    return slot + 1u >= (uint32_t)kMdFlush;
}

// position `g` (global) starts with the 3-byte prefix `pre`: walk its postings, compare the rest of each n-gram
// (-> true when one of its appends brought the CTA buffer to the flush threshold)
__device__ __noinline__ bool mdense_confirm(const MdenseParams &p, unsigned long long *sBuf, uint32_t *sN, uint32_t pre,
                                            int64_t g) {
    if (g < p.mp.own_lo || g >= p.mp.own_hi) return false;
    bool full = false;
    uint32_t slot = (pre * kGramMul) & p.mp.gtab_mask;
    for (;;) {
        const uint2 e = __ldg(p.mp.gtab + slot);
        if (e.y == 0u) return full;
        if (e.x == pre) {
            const uint32_t first = e.y & 0xFFFFFFu, cnt = e.y >> 24;
            for (uint32_t i = 0; i < cnt; i++) {
                const uint32_t post = __ldg(p.mp.postings + first + i);
                const uint32_t pid = post >> 8, j = post & 0xFFu;
                const BatchPat *bp = p.pats + pid;
                const int L = bp->L, s = (int)j * L;
                if (g + L > p.mp.N) continue;
                const uint8_t *t = p.mp.H + (g - p.mp.buf_lo);
                bool eq = true;
                for (int b = 3; b < L; b++)
                    if (__ldg(t + b) != bp->P[s + b]) {
                        eq = false;
                        break;
                    }
                if (eq) full |= mdense_append(p, sBuf, sN, (unsigned long long)(g - p.mp.buf_lo) | ((unsigned long long)j << 40) | ((unsigned long long)pid << 48));
            }
        }
        slot = (slot + 1) & p.mp.gtab_mask;
    }
}

__global__ void __launch_bounds__(kMultiThreads, 1)
k_filter_mdense(const __grid_constant__ MdenseParams p, int64_t nvec, int64_t ntiles) {
    extern __shared__ __align__(16) uint32_t mtbl[];
    unsigned long long *sBuf = reinterpret_cast<unsigned long long *>(mtbl + kMultiTblWords);
    uint32_t *sN = reinterpret_cast<uint32_t *>(sBuf + kMdBuf);
    __shared__ uint32_t sBase;
    for (int i = threadIdx.x; i < kMultiTblWords / 4; i += kMultiThreads)
        reinterpret_cast<uint4 *>(mtbl)[i] = __ldg(reinterpret_cast<const uint4 *>(p.mp.bits) + i);
    if (threadIdx.x == 0) *sN = 0;
    __syncthreads();
    const int lane = threadIdx.x & 31;
    const uint4 *base = reinterpret_cast<const uint4 *>(p.mp.H);
    for (int64_t t = blockIdx.x; t < ntiles; t += gridDim.x) {
        bool full = false;
#pragma unroll 1
        for (int u = 0; u < kMultiUnroll; u++) {
            const int64_t v = t * kMultiTileVecs + (int64_t)u * kMultiThreads + threadIdx.x;
            const uint4 d = (v < nvec) ? ldg_stream(base + v) : make_uint4(0, 0, 0, 0);
            uint32_t nx = __shfl_down_sync(0xFFFFFFFFu, d.x, 1);  // the 4 bytes after my 16
            if (lane == 31) nx = (v + 1 < nvec + 8) ? __ldg(reinterpret_cast<const uint32_t *>(base + v + 1)) : 0u;  // padded buffer
            const uint32_t ws[5] = {d.x, d.y, d.z, d.w, nx};
            uint32_t acc = 0;  // bit (15 - b) <-> position b of my vector
#pragma unroll
            for (int b = 0; b < 16; b++) {
                const uint32_t w = __funnelshift_r(ws[b >> 2], ws[(b >> 2) + 1], 8 * (b & 3)) & 0xFFFFFFu;
                const uint32_t h = multi_hash(w);
                acc = acc * 2u + ((mtbl[h >> 5] >> (h & 31u)) & 1u);
            }
            if (acc) {
                const int64_t off = v * 16;
                while (acc) {
                    const int bit = 31 - __clz(acc);
                    acc &= ~(1u << bit);
                    const int b = 15 - bit;
                    if (off + b + 3 > p.mp.buf_len) continue;
                    const uint32_t w = __funnelshift_r(ws[b >> 2], ws[(b >> 2) + 1], 8 * (b & 3)) & 0xFFFFFFu;
                    full |= mdense_confirm(p, sBuf, sN, w, p.mp.buf_lo + off + b);
                }
            }
        }
        // flush decision reduced inside the barrier from what happened before it (see k_lp_scan): warps that are a
        // tile ahead may already be appending again when a slower warp would read the count
        if (__syncthreads_or(full)) {
            flush_cta_buffer(sBuf, sN, min(*sN, (uint32_t)kMdBuf), &sBase, p.hits, p.hits_cap,
                             &p.mp.counters[CNT_MHITS], kMultiThreads);
            __syncthreads();
        }
    }
    __syncthreads();
    const uint32_t n = min(*sN, (uint32_t)kMdBuf);
    if (n) flush_cta_buffer(sBuf, sN, n, &sBase, p.hits, p.hits_cap, &p.mp.counters[CNT_MHITS], kMultiThreads);
}

// ------------------------------------------------------------------------------------------------
// On low-entropy haystacks (DNA) a 3-byte prefix hits about every 64th position, so the prefix scan is no filter.
//   k_filter_mdense2  finds the same hits with 2-bit keys: at EVERY position the 16-bit key of the 2-bit codes of the
//        8 symbols there (a 256-entry byte -> code table from the pass's four most frequent pattern bytes) indexes an
//        exact 64 Ki-bit table in shared memory; an n-gram shorter than 8 symbols is entered under every completion of
//        its key.  A flagged lane walks the key's postings (pattern, n-gram j) and compares ALL L bytes of n-gram j
//        with the text (bytes outside the four coded ones alias to code 0), appending exactly the hits k_filter_mdense
//        appends, for k_verify_mhits unchanged.  One launch scans [scan_lo, scan_hi) only: the host cuts the own range
//        into chunks whose hits fit the list, and verifies each chunk before scanning the next.
// ------------------------------------------------------------------------------------------------
constexpr int kHbKeySyms = 8;                                   // 2-bit key: codes of 8 symbols = 16 bits
constexpr int kHbKeyWords = 1 << (2 * kHbKeySyms - 5);          // 2048 words = 8 KiB, one bit per key
constexpr size_t kHbSmem2 = (size_t)kHbKeyWords * 4;
constexpr size_t kMdense2Smem = kHbSmem2 + (size_t)kMdBuf * 8 + 16;

// 2-bit codes of the 16 bytes of ws[0..3] and the 7 after them: symbol i at bits 2i and 2i+1
__device__ __forceinline__ unsigned long long key_codes(const uint8_t *sCode, const uint32_t (&ws)[6]) {
    unsigned long long codes = 0ull;
#pragma unroll
    for (int i = 0; i < 16 + kHbKeySyms - 1; i++)
        codes |= (unsigned long long)sCode[(ws[i >> 2] >> (8 * (i & 3))) & 0xFFu] << (2 * i);
    return codes;
}

struct Mdense2Params {
    MdenseParams dp;           // as for k_filter_mdense, gtab keyed by the 2-bit key (MdenseParams itself stays as
                               // k_verify_mhits takes it)
    int64_t scan_lo, scan_hi;  // global positions of this launch
    uint8_t code[256];         // byte -> 2-bit code
};

// position `g` (global, inside the scan and own ranges) carries `key`: walk its postings, compare each n-gram in full
// (-> true when one of its appends brought the CTA buffer to the flush threshold)
__device__ __noinline__ bool mdense2_confirm(const MdenseParams &p, unsigned long long *sBuf, uint32_t *sN, uint32_t key,
                                             int64_t g) {
    bool full = false;
    uint32_t slot = (key * kGramMul) & p.mp.gtab_mask;
    for (;;) {
        const uint2 e = __ldg(p.mp.gtab + slot);
        if (e.y == 0u) return full;
        if (e.x == key) {
            const uint32_t first = e.y & 0xFFFFFFu, cnt = e.y >> 24;
            for (uint32_t i = 0; i < cnt; i++) {
                const uint32_t post = __ldg(p.mp.postings + first + i);
                const uint32_t pid = post >> 8, j = post & 0xFFu;
                const BatchPat *bp = p.pats + pid;
                const int L = bp->L, s = (int)j * L;
                if (g + L > p.mp.N) continue;
                const uint8_t *t = p.mp.H + (g - p.mp.buf_lo);
                bool eq = true;
                for (int b = 0; b < L; b++)
                    if (__ldg(t + b) != bp->P[s + b]) {
                        eq = false;
                        break;
                    }
                if (eq) full |= mdense_append(p, sBuf, sN, (unsigned long long)(g - p.mp.buf_lo) | ((unsigned long long)j << 40) | ((unsigned long long)pid << 48));
            }
        }
        slot = (slot + 1) & p.mp.gtab_mask;
    }
}

// v0: the first 16-byte vector of the buffer this launch reads (the one holding scan_lo); nvec: vectors of the buffer
__global__ void __launch_bounds__(kMultiThreads, 1)
k_filter_mdense2(const __grid_constant__ Mdense2Params p, int64_t nvec, int64_t v0, int64_t ntiles) {
    extern __shared__ __align__(16) uint32_t md2_tbl[];
    unsigned long long *sBuf = reinterpret_cast<unsigned long long *>(md2_tbl + kHbKeyWords);
    uint32_t *sN = reinterpret_cast<uint32_t *>(sBuf + kMdBuf);
    __shared__ uint32_t sBase;
    __shared__ uint8_t sCode[256];
    const MdenseParams &dp = p.dp;
    for (int i = threadIdx.x; i < kHbKeyWords / 4; i += kMultiThreads)
        reinterpret_cast<uint4 *>(md2_tbl)[i] = __ldg(reinterpret_cast<const uint4 *>(dp.mp.bits) + i);
    for (int i = threadIdx.x; i < 256; i += kMultiThreads) sCode[i] = p.code[i];
    if (threadIdx.x == 0) *sN = 0;
    __syncthreads();
    const int lane = threadIdx.x & 31;
    const uint4 *base = reinterpret_cast<const uint4 *>(dp.mp.H);
    const int64_t lo = max(p.scan_lo, dp.mp.own_lo), hi = min(p.scan_hi, dp.mp.own_hi);  // positions that count
    for (int64_t t = blockIdx.x; t < ntiles; t += gridDim.x) {
        bool full = false;
#pragma unroll 1
        for (int u = 0; u < kMultiUnroll; u++) {
            const int64_t v = v0 + t * kMultiTileVecs + (int64_t)u * kMultiThreads + threadIdx.x;
            const uint4 d = (v < nvec) ? ldg_stream(base + v) : make_uint4(0, 0, 0, 0);
            uint32_t nx = __shfl_down_sync(0xFFFFFFFFu, d.x, 1);  // the 8 bytes after my 16
            uint32_t ny = __shfl_down_sync(0xFFFFFFFFu, d.y, 1);
            if (lane == 31 && v < nvec) {  // padded buffer
                const uint2 e = __ldg(reinterpret_cast<const uint2 *>(base + v + 1));
                nx = e.x;
                ny = e.y;
            }
            const uint32_t ws[6] = {d.x, d.y, d.z, d.w, nx, ny};
            const unsigned long long codes = key_codes(sCode, ws);
            uint32_t acc = 0;  // bit (15 - b) <-> position b of my vector
#pragma unroll
            for (int b = 0; b < 16; b++) {
                const uint32_t key = (uint32_t)(codes >> (2 * b)) & 0xFFFFu;
                acc = acc * 2u + ((md2_tbl[key >> 5] >> (key & 31u)) & 1u);
            }
            const int64_t g0 = dp.mp.buf_lo + v * 16;
            while (acc) {
                const int bit = 31 - __clz(acc);
                acc &= ~(1u << bit);
                const int b = 15 - bit;
                if (g0 + b < lo || g0 + b >= hi) continue;
                full |= mdense2_confirm(dp, sBuf, sN, (uint32_t)(codes >> (2 * b)) & 0xFFFFu, g0 + b);
            }
        }
        // flush decision reduced inside the barrier, as in k_filter_mdense
        if (__syncthreads_or(full)) {
            flush_cta_buffer(sBuf, sN, min(*sN, (uint32_t)kMdBuf), &sBase, dp.hits, dp.hits_cap,
                             &dp.mp.counters[CNT_MHITS], kMultiThreads);
            __syncthreads();
        }
    }
    __syncthreads();
    const uint32_t n = min(*sN, (uint32_t)kMdBuf);
    if (n) flush_cta_buffer(sBuf, sN, n, &sBase, dp.hits, dp.hits_cap, &dp.mp.counters[CNT_MHITS], kMultiThreads);
}

constexpr int kMhThreads = 128;
constexpr int kMhSlotBytes = 160;  // per-lane window slot: m + 2k + alignment slack (m <= 64, m + 2k + 8 <= 160)

template <bool REC>
__global__ void __launch_bounds__(kMhThreads)
k_verify_mhits(const __grid_constant__ MdenseParams p, RawRec *out, uint32_t cap, uint32_t *counters, const RecSet rs) {
    __shared__ __align__(16) uint8_t slots[kMhThreads][kMhSlotBytes];
    __shared__ __align__(16) uint8_t pats[kMhThreads][kBatchMaxM];
    const uint32_t nhits = counters[CNT_MHITS];
    if (nhits > p.hits_cap) {  // list overflowed: the host searches these patterns one by one
        if (blockIdx.x == 0 && threadIdx.x == 0) counters[CNT_OVERFLOW] = 1;
        return;
    }
    const int lane = threadIdx.x & 31;
    uint8_t *slot = slots[threadIdx.x];
    uint8_t *myP = pats[threadIdx.x];
    for (;;) {
        uint32_t base = 0;
        if (lane == 0) base = atomicAdd(&counters[CNT_MHITWORK], 32u);
        base = __shfl_sync(0xFFFFFFFFu, base, 0);
        if (base >= nhits) break;
        const uint32_t item = base + lane;
        bool valid = item < nhits;
        VerifyCtx c;
        c.H = p.mp.H;
        c.buf_lo = p.mp.buf_lo;
        c.buf_len = p.mp.buf_len;
        c.N = p.mp.N;
        c.own_lo = p.mp.own_lo;
        c.own_hi = p.mp.own_hi;
        c.m = c.k = 1;
        c.L = 1;
        c.n_ngrams = 1;
        int64_t idx = 0, alo = 0, lo = 0, hi = 0;
        int j = 0, tag = 0;
        if (valid) {
            const unsigned long long hv = p.hits[item];
            idx = p.mp.buf_lo + (int64_t)(hv & ((1ull << 40) - 1));
            j = (int)((hv >> 40) & 0xFFu);
            const uint32_t pid = (uint32_t)(hv >> 48);
            tag = (int)(pid << 8);
            const BatchPat *bp = p.pats + pid;
            c.m = bp->m;
            c.k = bp->k;
            c.L = bp->L;
            c.n_ngrams = bp->n_ngrams;
            for (int w = 0; w < kBatchMaxM / 4; w++)
                reinterpret_cast<uint32_t *>(myP)[w] = __ldg(reinterpret_cast<const uint32_t *>(bp->P) + w);
            if constexpr (REC) {  // the hit's own record; a hit on a separator is dropped
                valid = rec_bounds(rs, idx, lo, hi);
                if (valid) alo = stage_lane_window(c, idx - (int64_t)j * c.L, slot, lo, hi);
            } else {
                alo = stage_lane_window(c, idx - (int64_t)j * c.L, slot);
            }
        }
        verify_anchor_lev<3, REC>(c, myP, nullptr, slot - alo, idx, valid, nullptr, out, cap, counters, j, j + 1, tag,
                                  lo, hi);
    }
    if (blockIdx.x == 0 && threadIdx.x == 0) atomicAdd(&counters[CNT_CAND], nhits);
}

// ------------------------------------------------------------------------------------------------
// The LP-route patterns (m // (k+1) < 3) of a batch share a scan as well, 64 at a time.  The two necessary conditions
// of k_lp_scan -- first character in P[:k+1], and at least m-k characters of the window H[s : s+m+k) that occur in P
// -- are evaluated for ALL patterns at once with BIT-SLICED counters: a 256-entry table gives, per byte, the 64-bit
// vectors A (bit p: the byte occurs in pattern p) and F (bit p: it occurs in P_p[:k_p+1]); six 64-bit words hold, bit
// position p, the 6-bit number  (32 - need_p) + #{bytes of the sliding window in pattern p's set},  so bit-slice 5
// IS the vector "count_p >= need_p".  Sliding the window by one position adds the entering byte's A and removes the
// leaving byte's with one ripple over the six slices.  The window is the LONGEST m+k of the pass (a superset for the
// shorter patterns: still necessary); k_lp_verify_multi re-tests each survivor with its own pattern's exact window
// before running the bit-parallel automaton and, on acceptance, the literal simulation -- all per lane.
//   k_lp_scan_multi    CTA tile = 256 threads x 128 positions staged in shared memory (padded: conflict-free walks);
//                      survivors (pattern, start) buffered per CTA, one global atomic per flush.
//   k_lp_verify_multi  one survivor per thread.
// ------------------------------------------------------------------------------------------------
constexpr int kLmThreads = 256;
constexpr int kLmRun = 128;                         // positions a thread walks
constexpr int kLmTile = kLmThreads * kLmRun;        // 32768
constexpr int kLmHalo = 64;                         // >= longest window
constexpr int kLmBuf = 6144;
constexpr int kLmFlush = 2048;
constexpr size_t kLmTileBytes = ((size_t)(kLmTile + kLmHalo) / 128 * 132 + 132 + 15) / 16 * 16;  // padded tile, 16-aligned
constexpr size_t kLmSmem = kLmTileBytes + 256 * 16 + (size_t)kLmBuf * 8 + 16;
enum { CNT_LMLIST = 7, CNT_LMWORK = 8 };

struct LpMultiParams {
    const uint8_t *H;
    int64_t buf_lo, buf_len, N, own_lo, own_hi;   // own range = this chunk of starts
    const ulonglong2 *lut;                         // per byte: x = A vector, y = F vector
    unsigned long long bias[6];                    // bit slices of (32 - need_p)
    int wmax;                                      // longest m + k of the pass
    const BatchPat *pats;
    const uint32_t *pm32;                          // per pattern: 256 match masks {j : P[j] == c} (k_lp_verify_multi)
    unsigned long long *list;                      // (start - buf_lo) | pattern << 40: buffer-relative, so
                                                   // buf_len < 2^40 (check_shard)
    uint32_t list_cap;
    uint32_t *counters;
};

__device__ __forceinline__ uint32_t lm_addr(uint32_t i) { return i + 4u * (i >> 7); }  // 128-byte runs 132 bytes apart

__global__ void __launch_bounds__(kLmThreads)
k_lp_scan_multi(const __grid_constant__ LpMultiParams p) {
    extern __shared__ __align__(16) uint8_t lm_smem[];
    uint8_t *sH = lm_smem;
    ulonglong2 *sLut = reinterpret_cast<ulonglong2 *>(lm_smem + kLmTileBytes);
    unsigned long long *sBuf = reinterpret_cast<unsigned long long *>(sLut + 256);
    uint32_t *sN = reinterpret_cast<uint32_t *>(sBuf + kLmBuf);
    __shared__ uint32_t sBase;
    for (int i = threadIdx.x; i < 256; i += kLmThreads) sLut[i] = p.lut[i];
    if (threadIdx.x == 0) *sN = 0;
    __syncthreads();
    const int64_t hi = min(p.own_hi, p.N);                  // starts are < hi
    const int64_t lim = min(p.N, p.buf_lo + p.buf_len);     // bytes at or beyond this belong to no pattern's set
    const int64_t base = p.own_lo & ~(int64_t)127;          // tiles start on 128-byte boundaries (aligned word loads)
    const int64_t ntiles = hi > base ? (hi - base + kLmTile - 1) / kLmTile : 0;
    const int wmax = p.wmax;
    for (int64_t t = blockIdx.x; t < ntiles; t += gridDim.x) {
        const int64_t tile_lo = base + t * kLmTile;
        __syncthreads();  // the previous tile is consumed
        {   // stage [tile_lo, tile_lo + kLmTile + kLmHalo) : coalesced 4-byte loads into the padded layout
            const int nwords = (kLmTile + kLmHalo) / 4;
            const uint8_t *src = p.H + (tile_lo - p.buf_lo);  // (may point before the buffer: guarded below)
            const int64_t first = p.buf_lo - tile_lo;                  // bytes of the tile before the buffer
            const int64_t avail = p.buf_lo + p.buf_len + 128 - tile_lo;  // readable bytes (padded buffer)
            for (int w = threadIdx.x; w < nwords; w += kLmThreads) {
                const int64_t b = (int64_t)w * 4;
                const uint32_t v = (b >= first && b + 4 <= avail) ? __ldg(reinterpret_cast<const uint32_t *>(src + b)) : 0u;
                *reinterpret_cast<uint32_t *>(sH + lm_addr((uint32_t)w * 4u)) = v;
            }
        }
        __syncthreads();
        const uint32_t r0 = threadIdx.x * kLmRun;            // my run inside the tile
        const int64_t s0 = tile_lo + r0;
        unsigned long long C[6];
#pragma unroll
        for (int i = 0; i < 6; i++) C[i] = p.bias[i];
        for (int j = 0; j < wmax; j++) {                      // count over [s0, s0 + wmax)
            unsigned long long carry = (s0 + j < lim) ? sLut[sH[lm_addr(r0 + j)]].x : 0ull;
#pragma unroll
            for (int i = 0; i < 6; i++) {
                const unsigned long long c = C[i];
                C[i] = c ^ carry;
                carry &= c;
            }
        }
        for (int r = 0; r < kLmRun; r++) {
            const int64_t s = s0 + r;
            ulonglong2 lf = make_ulonglong2(0ull, 0ull);
            if (s < lim) lf = sLut[sH[lm_addr(r0 + r)]];
            unsigned long long surv = C[5] & lf.y;            // count_p >= need_p  and  first character of p
            if (surv && s >= p.own_lo && s < hi) {
                const uint32_t n = (uint32_t)__popcll(surv);
                uint32_t slot = atomicAdd(sN, n);
                while (surv) {
                    const int pid = __ffsll((long long)surv) - 1;
                    surv &= surv - 1;
                    const unsigned long long ent = (unsigned long long)(s - p.buf_lo) | ((unsigned long long)pid << 40);
                    if (slot < (uint32_t)kLmBuf) {
                        sBuf[slot] = ent;
                    } else {  // CTA buffer full: straight to the list
                        const uint32_t g = atomicAdd(&p.counters[CNT_LMLIST], 1u);
                        if (g < p.list_cap) p.list[g] = ent;
                    }
                    slot++;
                }
            }
            // slide: the byte at s leaves, the byte at s + wmax enters
            const unsigned long long ae = (s + wmax < lim) ? sLut[sH[lm_addr(r0 + r + wmax)]].x : 0ull;
            unsigned long long up = ae & ~lf.x, dn = lf.x & ~ae;
#pragma unroll
            for (int i = 0; i < 6; i++) {
                const unsigned long long c = C[i];
                C[i] = c ^ up ^ dn;
                up &= c;
                dn &= ~c;
            }
        }
        __syncthreads();
        const uint32_t n = min(*sN, (uint32_t)kLmBuf);
        // (the barrier at the top of the next tile orders the reset before the next append)
        if (n >= (uint32_t)kLmFlush)
            flush_cta_buffer(sBuf, sN, n, &sBase, p.list, p.list_cap, &p.counters[CNT_LMLIST], kLmThreads);
    }
    __syncthreads();
    const uint32_t n = min(*sN, (uint32_t)kLmBuf);
    if (n) flush_cta_buffer(sBuf, sN, n, &sBase, p.list, p.list_cap, &p.counters[CNT_LMLIST], kLmThreads);
}

// Between scan and verification: k_lm_refine applies each survivor's OWN window (the scan used the longest one of the
// pass) and keeps the exact survivors, counting them per pattern; k_lm_scatter then groups them by pattern (counting
// sort), so that the lanes of a warp of k_lp_verify_multi run the automaton of the SAME pattern (same m, k, loop
// bounds) almost always.
constexpr int kLmSortThreads = 256;

__global__ void __launch_bounds__(kLmSortThreads)
k_lm_refine(const __grid_constant__ LpMultiParams p, unsigned long long *kept, uint32_t *hist /* [64] + kept count at [64] */) {
    __shared__ uint32_t sHist[64];
    __shared__ unsigned long long sKeep[kLmSortThreads];
    __shared__ unsigned long long sA[256];  // per byte: bit p = the byte occurs in pattern p
    __shared__ uint32_t sN, sBase;
    const uint32_t n = p.counters[CNT_LMLIST];
    if (n > p.list_cap) return;  // overflow: k_lp_verify_multi reports it
    for (int i = threadIdx.x; i < 256; i += kLmSortThreads) sA[i] = p.lut[i].x;
    const uint8_t *W = p.H - p.buf_lo;
    const int64_t lim = min(p.N, p.buf_lo + p.buf_len);
    if (threadIdx.x < 64) sHist[threadIdx.x] = 0;
    for (uint32_t base = blockIdx.x * kLmSortThreads; base < n; base += gridDim.x * kLmSortThreads) {
        if (threadIdx.x == 0) sN = 0;
        __syncthreads();
        const uint32_t i = base + threadIdx.x;
        if (i < n) {
            const unsigned long long ent = p.list[i];
            const int64_t st = p.buf_lo + (int64_t)(ent & ((1ull << 40) - 1));
            const uint32_t pid = (uint32_t)(ent >> 40);
            const BatchPat *bp = p.pats + pid;
            const int m = bp->m, k = bp->k, win = m + k, need = m - k;
            int cnt = 0;
            for (int j = 0; j < win && st + j < lim; j++) cnt += (int)((sA[W[st + j]] >> pid) & 1ull);
            if (cnt >= need) {
                sKeep[atomicAdd(&sN, 1u)] = ent;
                atomicAdd(&sHist[pid], 1u);
            }
        }
        __syncthreads();
        const uint32_t kn = sN;
        if (kn) {
            if (threadIdx.x == 0) sBase = atomicAdd(&hist[64], kn);
            __syncthreads();
            if (threadIdx.x < kn) kept[sBase + threadIdx.x] = sKeep[threadIdx.x];
        }
        __syncthreads();
    }
    __syncthreads();
    if (threadIdx.x < 64 && sHist[threadIdx.x]) atomicAdd(&hist[threadIdx.x], sHist[threadIdx.x]);
}

// kept[0 .. hist[64]) -> sorted[...] grouped by pattern; cursors[64] start at zero
__global__ void __launch_bounds__(kLmSortThreads)
k_lm_scatter(const unsigned long long *kept, const uint32_t *hist, uint32_t *cursors, unsigned long long *sorted) {
    __shared__ uint32_t sOff[64], sCnt[64], sBase[64];
    const uint32_t n = hist[64];
    if (threadIdx.x == 0) {
        uint32_t acc = 0;
        for (int q = 0; q < 64; q++) {
            sOff[q] = acc;
            acc += hist[q];
        }
    }
    for (uint32_t base = blockIdx.x * kLmSortThreads; base < n; base += gridDim.x * kLmSortThreads) {
        if (threadIdx.x < 64) sCnt[threadIdx.x] = 0;
        __syncthreads();
        const uint32_t i = base + threadIdx.x;
        unsigned long long ent = 0;
        uint32_t pid = 0, rank = 0;
        if (i < n) {
            ent = kept[i];
            pid = (uint32_t)(ent >> 40);
            rank = atomicAdd(&sCnt[pid], 1u);
        }
        __syncthreads();
        if (threadIdx.x < 64 && sCnt[threadIdx.x]) sBase[threadIdx.x] = atomicAdd(&cursors[threadIdx.x], sCnt[threadIdx.x]);
        __syncthreads();
        if (i < n) sorted[sOff[pid] + sBase[pid] + rank] = ent;
        __syncthreads();
    }
}

struct LpLaneCtx {  // what sim_lev_lp needs
    int32_t m, k;
    int64_t N;
};

// One survivor per LANE, with refill: the automata of different survivors die after very different numbers of
// characters, so a lane whose survivor is finished fetches the next one (warp-aggregated atomic on a work counter)
// instead of idling until the slowest of its 31 neighbours is done -- every iteration of the loop is one automaton
// step for (almost) all lanes.  An accepting lane runs the literal simulation (rare) and goes back to the pool.
enum { CNT_LMNEXT = 10 };

// REC: c.N is the end of the survivor's own record, and a start on a separator opens nothing (as in k_lp_verify).
template <int K, bool REC>
__global__ void __launch_bounds__(kLpThreads)
k_lp_verify_multi(const __grid_constant__ LpMultiParams p, const unsigned long long *sorted, const uint32_t *hist,
                  uint32_t *scratch, int cap, RawRec *out, uint32_t ocap, uint32_t *counters, const RecSet rs) {
    __shared__ __align__(4) uint8_t sPat[kLpThreads][kBatchMaxM / 2];  // LP patterns are at most 31 bytes
    if (counters[CNT_LMLIST] > p.list_cap) {  // the scan's list overflowed: the host searches these patterns one by one
        if (blockIdx.x == 0 && threadIdx.x == 0) counters[CNT_LMWORK] = 1;
        return;
    }
    const uint32_t n = hist[64];  // exact survivors, grouped by pattern
    const int64_t tid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int lane = threadIdx.x & 31;
    uint32_t *A = scratch + tid * 2 * (int64_t)cap, *B = A + cap;
    const uint8_t *W = p.H - p.buf_lo;  // W[g]: byte at global position g
    uint8_t *myP = sPat[threadIdx.x];
    bool have = false, drained = false;
    int64_t st = 0, i = 0;
    uint32_t pid = 0;
    LpLaneCtx c;
    c.m = 2;
    c.k = 1;
    c.N = p.N;
    const uint32_t *pm = p.pm32;
    uint32_t R[K + 1];
#pragma unroll
    for (int d = 0; d <= K; d++) R[d] = 0;
    for (;;) {
        const unsigned want = __ballot_sync(0xFFFFFFFFu, !have && !drained);
        bool accept = false;
        if (want) {
            const int leader = __ffs(want) - 1;
            uint32_t base = 0;
            if (lane == leader) base = atomicAdd(&counters[CNT_LMNEXT], (uint32_t)__popc(want));
            base = __shfl_sync(0xFFFFFFFFu, base, leader);
            if (!have && !drained) {
                const uint32_t idx = base + (uint32_t)__popc(want & ((1u << lane) - 1u));
                if (idx >= n) {
                    drained = true;
                } else {
                    const unsigned long long ent = sorted[idx];
                    st = p.buf_lo + (int64_t)(ent & ((1ull << 40) - 1));
                    pid = (uint32_t)(ent >> 40);
                    const BatchPat *bp = p.pats + pid;
                    c.m = bp->m;
                    c.k = bp->k;
                    pm = p.pm32 + (size_t)pid * 256;
                    for (int w = 0; w < kBatchMaxM / 8; w++)
                        reinterpret_cast<uint32_t *>(myP)[w] = __ldg(reinterpret_cast<const uint32_t *>(bp->P) + w);
                    int j0 = -1;  // make_char2first_subseq_index (levenshtein.py:44-49)
                    const uint8_t ch = W[st];
                    for (int j = 0; j <= min(c.k, c.m - 1); j++)
                        if (myP[j] == ch) {
                            j0 = j;
                            break;
                        }
                    if constexpr (REC) {
                        int64_t lo;
                        if (!rec_bounds(rs, st, lo, c.N)) j0 = -1;
                    }
                    if (j0 >= 0) {
                        if (j0 + 1 == c.m) {
                            accept = true;  // :78-79
                        } else {
#pragma unroll
                            for (int d = 0; d <= K; d++) R[d] = (d == j0) ? (1u << (j0 + 1)) : 0u;  // :80-81
                            i = st + 1;
                            have = true;
                        }
                    }
                }
            }
        }
        if (__all_sync(0xFFFFFFFFu, drained && !have && !accept)) break;
        if (have) {  // one character
            if (i >= (REC ? c.N : p.N)) {
                accept = lp_nfa_end<K>(R, c.m, c.k);
                have = false;
            } else {
                bool alive = true;
                if (lp_nfa_step<K>(R, __ldg(pm + W[i]), i + 1 < (REC ? c.N : p.N), c.m, c.k, alive)) {
                    accept = true;
                    have = false;
                } else if (!alive) {
                    have = false;
                }
                i++;
            }
        }
        if (accept) {  // this start emits something: the literal simulation produces the records (with multiplicities)
            if (!sim_lev_lp(c, myP, W, st, A, B, cap, out, ocap, counters, 1 | (int)(pid << 8)))
                atomicExch(&counters[CNT_OVERFLOW], 1u);
        }
    }
    if (blockIdx.x == 0 && threadIdx.x == 0) atomicAdd(&counters[CNT_CAND], counters[CNT_LMLIST]);
}

constexpr int kVmThreads = 128;

// REC (here and in the other batch verify kernels): the handle holds a record set `rs` (DESIGN.md section 5.11); each
// anchor or start is verified inside its own record, as the single-pattern kernels do.  The REC == false
// instantiations never read rs.
template <bool REC>
__global__ void __launch_bounds__(kVmThreads)
k_verify_multi(const __grid_constant__ MultiParams p, const BatchPat *pats, RawRec *out, uint32_t cap, uint32_t *counters,
               const RecSet rs) {
    __shared__ __align__(8) uint8_t sPall[kVmThreads / 32][kBatchMaxM];
    __shared__ unsigned long long sPMall[kVmThreads / 32][256];
    __shared__ uint32_t sWinAll[kVmThreads / 32][kWinWords];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    uint8_t *sP = sPall[warp];
    unsigned long long *sPM = sPMall[warp];
    uint32_t *sWin = sWinAll[warp];
    const uint32_t nitems = min(counters[CNT_GRAN], p.work_cap);
    uint32_t cur_pid = 0xFFFFFFFFu;
    VerifyCtx c;
    c.H = p.H;
    c.buf_lo = p.buf_lo;
    c.buf_len = p.buf_len;
    c.N = p.N;
    c.own_lo = p.own_lo;
    c.own_hi = p.own_hi;
    c.m = c.k = c.L = c.n_ngrams = 0;
    for (;;) {
        uint32_t item = 0;
        if (lane == 0) item = atomicAdd(&counters[CNT_WORK], 1u);
        item = __shfl_sync(0xFFFFFFFFu, item, 0);
        if (item >= nitems) break;
        const WorkItem it = p.work[item];
        if (it.pid != cur_pid) {  // load the pattern and build its match table (PM[c] = {i : P[i] == c})
            const BatchPat *bp = pats + it.pid;
            __syncwarp();
            if (lane < kBatchMaxM / 4) reinterpret_cast<uint32_t *>(sP)[lane] = reinterpret_cast<const uint32_t *>(bp->P)[lane];
            for (int ch = lane; ch < 256; ch += 32) sPM[ch] = 0ull;
            c.m = bp->m;
            c.k = bp->k;
            c.L = bp->L;
            c.n_ngrams = bp->n_ngrams;
            __syncwarp();
            for (int i = lane; i < c.m; i += 32) atomicOr(&sPM[sP[i]], 1ull << i);
            __syncwarp();
            cur_pid = it.pid;
        }
        verify_granule_lev<1, REC>(c, sP, sPM, sWin, (int64_t)it.granule, lane, nullptr, out, cap, counters,
                                   (int)(it.pid << 8), rs);
        if (lane == 0) p.set[it.slot] = 0ull;  // the set is empty again when the kernel ends
    }
    if (blockIdx.x == 0 && threadIdx.x == 0) atomicAdd(&counters[CNT_CAND], nitems);
}

}  // namespace fzb
