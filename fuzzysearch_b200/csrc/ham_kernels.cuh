// ham_kernels.cuh -- substitutions-only (Hamming) search: every start p in [0, N-m] with
// Hamming(P, H[p:p+m]) <= k  (substitutions_only.py:37-215 == brute force, SURVEY F13).
//
// k_hamming_count -- the HBM-streaming kernel (used when m >= 4k+7 and k <= 7):
//   Counting q-sample filter.  An occurrence at p contains W = floor((m-3)/4) four-byte-aligned words
//   (at ANY alignment of p); a substitution spoils at most one of them, so at least Wc-k of the first
//   Wc = min(W, 8) aligned words inside it equal the pattern 4-gram at their own offset.  Unlike the
//   Levenshtein filter a single q-gram hit is not selective on small alphabets (DNA: 29 grams among
//   256 possible words), so the kernel COUNTS: per alignment class o0 = (first aligned word) - p in
//   {0,1,2,3} it keeps Wc counters, one per occurrence whose counted words are still being read, and
//   every aligned text word w adds 1 to the counters whose current pattern 4-gram equals w.  The 32
//   counters of the four classes are bit-sliced (ham_recur.h): one register per bit of the counters, and
//   the table entry of hash(w) is the 32 match bits, bit 8*o0 + i <-> w == P[o0+4i : o0+4i+4) -- one
//   LDS.32 per text word, replicated per lane (bank = lane: conflict-free).  The carry out of the top
//   slice flags the word at which an occurrence's (Wc-k)-th counted word matched.  Two slices count
//   to 4 and serve thresholds Wc-k <= 4; three count to 8.
//   The recurrence runs ALONG the text, so each thread owns one 128-byte row of a tile; tiles are
//   staged global -> shared by TMA (cp.async.bulk.tensor.2d, SWIZZLE_128B so that the per-thread
//   row reads are bank-conflict free, mbarrier complete_tx, 2-stage ring), one elected thread issuing.
//   Flagged rows (rare: true near-matches) are re-checked exactly, position by position.
// k_hamming_scan  -- brute-force fallback for short patterns / large k.
#pragma once
#include <cuda.h>

#include "ham_recur.h"
#include "kernels.cuh"

namespace fzb {

constexpr int kHamThreads = 256;

// Mismatches between the text bytes text(0 .. m-1) and sP[0 .. m-1]; counting stops once they exceed k.
template <class Text>
__device__ __forceinline__ int ham_mismatches(Text text, const uint8_t *sP, int m, int k) {
    int nd = 0;
    for (int i = 0; i < m; i++) {
        nd += (text(i) != sP[i]);
        if (nd > k) break;
    }
    return nd;
}

// REC: does the occurrence [pos, pos + m) lie inside one record of `rs`?  (Asked of the few starts that pass the
// mismatch count only.)
template <bool REC>
__device__ __forceinline__ bool ham_in_record(const RecSet &rs, int64_t pos, int m) {
    if (!REC) return true;
    int64_t lo, hi;
    return rec_bounds(rs, pos, lo, hi) && pos + m <= hi;
}

template <bool REC>
__global__ void __launch_bounds__(kHamThreads)
k_hamming_scan(const ScanParams p, RawRec *out, uint32_t cap, uint32_t *counters, const RecSet rs) {
    __shared__ uint8_t sP[256];
    for (int i = threadIdx.x; i < 256; i += blockDim.x) sP[i] = p.P[i];
    __syncthreads();
    const int m = p.m, k = p.k;
    const int64_t last = min(p.own_hi, p.N - m + 1);  // exclusive bound on starts
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t pos = p.own_lo + (int64_t)blockIdx.x * blockDim.x + threadIdx.x; pos < last; pos += stride) {
        const uint8_t *h = p.H + (pos - p.buf_lo);
        const int nd = ham_mismatches([&](int i) { return __ldg(h + i); }, sP, m, k);
        if (nd <= k && ham_in_record<REC>(rs, pos, m)) emit(out, cap, counters, pos, pos + m, pos, nd, 0);
    }
}

// ---- counting filter --------------------------------------------------------------------------------
constexpr int kHcThreads = 256;               // one 128-byte row per thread; 2 CTAs per SM
constexpr int kHcRowBytes = 128;
constexpr int kHcHaloRows = 8;                // one swizzle atom; only its last row is read
constexpr int kHcTileRows = kHcHaloRows + kHcThreads;            // 264
constexpr int kHcStageBytes = kHcTileRows * kHcRowBytes;         // 33792 (multiple of 1024)
constexpr int kHcStages = 2;
constexpr int kHcTableBytes = kHcBuckets * 32 * 4;               // 32 KiB: 32 replicas x 4 B per bucket
constexpr size_t kHcSmem = (size_t)kHcStages * kHcStageBytes + kHcTableBytes + 64;
struct HamCountParams {
    int Wc;        // counted words per occurrence (<= 8)
    int bias;      // 2^slices - (Wc - k): the counters' start value, so that they carry out at Wc - k matches
    int64_t nrows; // rows of the buffer that hold data: ceil(buf_len / 128)
};

// swizzled shared address of 16-byte chunk j of local row r (SWIZZLE_128B: chunk index ^= row % 8)
__device__ __forceinline__ uint32_t hc_chunk(uint32_t stage, int r, int j) {
    return stage + r * kHcRowBytes + ((j ^ (r & 7)) << 4);
}

// SLICES = 2 (thresholds Wc - k <= 4) or 3: the bit slices of the counters (ham_recur.h).
template <int SLICES>
__global__ void __launch_bounds__(kHcThreads, 2)
k_hamming_count(const ScanParams p, const HamCountParams hp, const __grid_constant__ CUtensorMap map256,
                const __grid_constant__ CUtensorMap map8) {
    extern __shared__ __align__(1024) uint8_t hc_smem[];  // SWIZZLE_128B tiles need 1024-byte alignment
    uint8_t *base = hc_smem;
    uint32_t *table = reinterpret_cast<uint32_t *>(base + kHcStages * kHcStageBytes);
    uint64_t *full = reinterpret_cast<uint64_t *>(base + kHcStages * kHcStageBytes + kHcTableBytes);
    const int tid = threadIdx.x, lane = tid & 31;
    const int Wc = hp.Wc;

    // bucket b, replica r (= lane): word b * 32 + r; bit 8 * o0 + i <-> w == P[o0+4i : o0+4i+4)
    for (int i = tid; i < kHcBuckets * 32; i += kHcThreads) table[i] = 0u;
    if (tid == 0) {
        for (int s = 0; s < kHcStages; s++) mbar_init(&full[s], 1);
        mbar_init_fence();
    }
    __syncthreads();
    if (tid < 32) {  // replica `tid` of the table: add the pattern's 4-grams (serial per replica: no races)
        for (int o0 = 0; o0 < 4; o0++)
            for (int i = 0; i < Wc; i++)  // each (class, field) pair exactly once
                table[hc_bucket(hc_gram(p.P, o0 + 4 * i)) * 32 + tid] |= 1u << (8 * o0 + i);
    }
    __syncthreads();

    const int64_t ntiles = (hp.nrows + kHcThreads - 1) / kHcThreads;
    const uint32_t B0 = (hp.bias & 1) ? 0x01010101u : 0u, B1 = (hp.bias & 2) ? 0x01010101u : 0u,
                   B2 = (hp.bias & 4) ? 0x01010101u : 0u;
    auto issue = [&](int64_t tile, int s) {  // one elected thread: 264 rows = 8 (halo atom) + 256
        const int r0 = (int)(tile * kHcThreads) - kHcHaloRows;
        uint8_t *dst = base + s * kHcStageBytes;
        mbar_expect_tx(&full[s], kHcStageBytes);
        tma_load_2d(dst, &map8, 0, r0, &full[s]);
        tma_load_2d(dst + kHcHaloRows * kHcRowBytes, &map256, 0, r0 + kHcHaloRows, &full[s]);
    };
    int64_t tile = blockIdx.x;
    if (tid == 0) {
        if (tile < ntiles) issue(tile, 0);
        if (tile + gridDim.x < ntiles) issue(tile + gridDim.x, 1);
    }
    const uint32_t my_table = smem_u32(table) + (lane << 2);  // my replica of the table: bank = lane
    const uint32_t stage0 = smem_u32(base);
    uint32_t phases = 0;  // bit s = parity to wait for on stage s
    for (int it = 0; tile < ntiles; tile += gridDim.x, it++) {
        const int s = it & 1;
        mbar_wait(&full[s], (phases >> s) & 1u);
        phases ^= 1u << s;
        const uint32_t st = stage0 + s * kHcStageBytes;
        const int r = kHcHaloRows + tid;
        HamSliced cnt{0u, 0u, 0u};
        HamSliced2 cnt2{0u, 0u};
        uint32_t acc = 0;
#define HS_STEP(WORD, track)                                                                 \
    {                                                                                        \
        const uint32_t M = lds32(my_table + (hc_bucket(WORD) << 7));                         \
        const uint32_t c = SLICES == 2 ? ham_sliced2_step(cnt2, M, B0, B1)                   \
                                       : ham_sliced_step(cnt, M, B0, B1, B2);                \
        if (track) acc |= c;                                                                 \
    }
        {  // warm-up: the last 7 words of the previous row (their candidates belong to that row's thread)
            const uint4 a = lds128(hc_chunk(st, r - 1, 6)), b = lds128(hc_chunk(st, r - 1, 7));
            HS_STEP(a.y, false) HS_STEP(a.z, false) HS_STEP(a.w, false)
            HS_STEP(b.x, false) HS_STEP(b.y, false) HS_STEP(b.z, false) HS_STEP(b.w, false)
        }
#pragma unroll
        for (int j = 0; j < 8; j++) {
            const uint4 d = lds128(hc_chunk(st, r, j));
            HS_STEP(d.x, true) HS_STEP(d.y, true) HS_STEP(d.z, true) HS_STEP(d.w, true)
        }
#undef HS_STEP
        if (acc) {
            // some start passed the filter at a word of my row (rare: true near-matches): mark its granules;
            // k_verify_ham re-checks them exactly.  The counters fire at the word of the (Wc-k)-th match,
            // anywhere from the first to the last counted word of the occurrence.
            const int64_t grow = tile * kHcThreads + tid;  // buffer row index
            const int64_t pr_lo = 4 * (grow * 32 - Wc + 1) - 3;
            const int64_t pr_hi = 4 * (grow * 32 + 31);
            mark_range_inline(p, p.buf_lo + max(pr_lo, (int64_t)0), p.buf_lo + pr_hi);
        }
        __syncthreads();  // everyone is done with stage s
        if (tid == 0 && tile + 2 * (int64_t)gridDim.x < ntiles) issue(tile + 2 * (int64_t)gridDim.x, s);
    }
}

// ---- exact verification of the marked granules (same work-list scheme as k_verify_lev) -------------
template <bool REC>
__device__ __forceinline__ void verify_granule_ham(const ScanParams &p, const uint8_t *sP, uint32_t *sWin,
                                                   int64_t granule, int lane, RawRec *out, uint32_t cap,
                                                   uint32_t *counters, const RecSet &rs) {
    const int m = p.m, k = p.k;
    const int64_t gbase = p.buf_lo + (granule << kGranuleShift);
    const int64_t alo = stage_window(p, gbase, m, lane, sWin);
    const uint8_t *W = reinterpret_cast<const uint8_t *>(sWin) - alo;
#pragma unroll 1
    for (int half = 0; half < kGranule / 32; half++) {
        const int64_t pos = gbase + half * 32 + lane;
        if (pos < p.own_lo || pos >= p.own_hi || pos + m > p.N) continue;
        const int nd = ham_mismatches([&](int i) { return W[pos + i]; }, sP, m, k);
        if (nd <= k && ham_in_record<REC>(rs, pos, m)) emit(out, cap, counters, pos, pos + m, pos, nd, 0);
    }
}

template <bool REC>
__global__ void __launch_bounds__(kVerifyThreads)
k_verify_ham(const ScanParams p, uint64_t bitmap_words, const uint32_t *glist, uint32_t glist_cap, int scan_mode,
             RawRec *out, uint32_t cap, uint32_t *counters, const RecSet rs) {
    __shared__ uint8_t sP[256];
    __shared__ uint32_t sWinAll[kVerifyThreads / 32][kWinWords];
    for (int i = threadIdx.x; i < 256; i += blockDim.x) sP[i] = p.P[i];
    __syncthreads();
    const int lane = threadIdx.x & 31;
    uint32_t *sWin = sWinAll[threadIdx.x >> 5];
    for_each_marked_granule(p.bitmap, bitmap_words, glist, glist_cap, scan_mode, counters, [&](int64_t g) {
        verify_granule_ham<REC>(p, sP, sWin, g, lane, out, cap, counters, rs);
    });
}

}  // namespace fzb
