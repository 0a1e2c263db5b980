// nearest_kernels.cuh -- fzb_nearest_distance / fzb_nearest_per_record (DESIGN.md section 5.14): the smallest
// Levenshtein distance of the pattern to any substring of the sequence, without a distance limit.
//
// E(e) = min over s <= e of lev(P, S[s:e]) is the bottom row of Sellers' table with a free start (D[0][j] = 0).
// k_nearest_scan runs its bit-vector form (Myers 1999, Hyyro 2003): the column is kept as the vertical deltas Pv / Mv,
// one bit per pattern symbol, and the score follows the horizontal delta at bit m - 1.  Nothing is shifted into the
// horizontal deltas (the search form; expand_bp in kernels.cuh is the prefix-anchored form, which shifts +1 in).
//
// Parallel along the text.  A thread owns a segment [a, b) of the text and first runs the recurrence, untracked, over
// the 2m bytes before a, from the initial column (Pv all ones, score m).  That is exact, not a heuristic: a column
// started at w computes E_w(e) = min over w <= s <= e, and for e >= w + 2m the two agree -- E(e) <= m (the empty
// substring), and a substring at distance d <= m from P is at most m + d <= 2m long, so some optimal s is >= e - 2m >= w.
// Each later score depends on the text only through these minima, so every score the thread records is E itself.
//
// The text is read straight from global memory, 16 bytes per load and lane (the lines of a lane's segment stay in L1
// between its loads); a segment is `seg` bytes, 512 to 4 096, chosen by the host from the sequence length.  The
// match masks PM[c] sit in shared memory.  With one word (m <= 64) the table is replicated per lane, entry
// c * 32 + lane: a 32-bit entry falls into bank `lane`, a 64-bit entry into banks 2 lane and 2 lane + 1 of its half
// warp, so 32 lanes looking up 32 different bytes never share a bank with different addresses (no conflict for any
// text).  With 2 to 4 words (m <= 255, correct but not tuned) one table [c][word] serves all lanes.
//
// Results.  Whole sequence: a thread keeps (minimum, ends at the minimum, first such end); warps, then the CTA combine
// them, and the CTA sends one atomicMin of dist << 48 | first_end and stores (minimum, count) as its partial;
// k_nearest_count adds the counts of the partials at the global minimum.  All of it is min / integer addition: the
// answer does not depend on thread, CTA or launch order.  Record sets (REC): the column is reset at every record
// start, a thread finds its first record as rec_bounds does and walks the offsets as its segment crosses separators, and
// each (record, thread) sends one atomicMin of dist << 32 | end - record start into the record's word, which
// k_nearest_fill set to the empty record's (m, 0).  The end position 0 (score m) is that initial value in both forms.
#pragma once
#include "common.cuh"
#include "best_kernels.cuh"

namespace fzb {

constexpr int kNearThreads = 256;
constexpr int kNearMinSeg = 512, kNearMaxSeg = 4096;  // bytes per thread (multiples of 16)
constexpr int kNearMaxGrid = 1024;                    // CTAs of a scan (partials of the whole-sequence form)
constexpr uint64_t kNearNoEnd = (1ull << 48) - 1;

struct NearParams {
    const uint8_t *H;
    int64_t N;
    int32_t m, seg;
    uint64_t *result;   // [0] dist << 48 | first_end, [1] n_ends
    uint64_t *partial;  // per CTA: its minimum, its count of ends there
    uint64_t *words;    // REC: dist << 32 | end per record
    uint8_t P[256];
};

template <int BITS> struct NearWord { typedef uint64_t type; };
template <> struct NearWord<32> { typedef uint32_t type; };

__host__ __device__ constexpr int near_words(int bits) { return bits <= 64 ? 1 : bits / 64; }
// resident CTAs per SM of a nearest kernel of word width `bits`: its __launch_bounds__ and the host's grids
__host__ __device__ constexpr int near_ctas_per_sm(int bits) { return bits == 32 ? 4 : bits == 64 ? 3 : 2; }
__host__ __device__ constexpr size_t near_smem(int bits) { return bits <= 64 ? (size_t)256 * 32 * (bits / 8) : (size_t)256 * (bits / 8); }

__global__ void k_nearest_fill(uint64_t *words, uint64_t n, uint64_t value) {
    const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) words[i] = value;
}

// (minimum, ends at the minimum, first such end) of two disjoint sets of end positions
__device__ __forceinline__ void near_merge(uint32_t &best, uint64_t &cnt, uint64_t &first, uint32_t ob, uint64_t oc,
                                           uint64_t of) {
    if (ob < best) {
        best = ob;
        cnt = oc;
        first = of;
    } else if (ob == best) {
        cnt += oc;
        if (of < first) first = of;
    }
}

template <int BITS>
struct NearCol {  // one column of the table and what the thread has seen of its bottom row
    typedef typename NearWord<BITS>::type word;
    static constexpr int NW = near_words(BITS);
    word Pv[NW], Mv[NW];
    uint32_t score, top;          // top: the bit of row m - 1 in the last word
    uint32_t best, cnt, first;    // tracked ends: the minimum below m (else m), its count, the first (as `rel`)
    const word *pm;               // this lane's view of the table

    // what the shared scans ask of a column: the best before any end (the end position 0 scores m), whether a
    // best is worth reporting (the end position 0 is the prefill's), and how many bytes before a segment make it exact
    static __device__ __forceinline__ uint32_t none(uint32_t m) { return m; }
    static __device__ __forceinline__ bool has(uint32_t best, uint32_t m) { return best < m; }
    static __device__ __forceinline__ int64_t warm(uint32_t m) { return 2 * (int64_t)m; }

    __device__ __forceinline__ void reset(uint32_t m) {
#pragma unroll
        for (int w = 0; w < NW; w++) {
            Pv[w] = ~(word)0;
            Mv[w] = 0;
        }
        score = best = m;
        cnt = 0;
        first = 0;
    }

    // the column behind text byte c; rel: the end position it closes, relative to the caller's base.  HIN: the
    // horizontal delta of row 0 -- 0 in the search form (D[0][j] = 0), +1 in the prefix-anchored form (D[0][j] = j)
    template <bool TRACK, int HIN = 0>
    __device__ __forceinline__ void step(uint32_t c, uint32_t rel) {
        int hin = HIN;
#pragma unroll
        for (int w = 0; w < NW; w++) {
            word Eq = NW == 1 ? pm[c * 32] : pm[c * NW + w];
            const word pv = Pv[w], mv = Mv[w];
            const word Xv = Eq | mv;
            if (NW > 1) Eq |= (word)(hin < 0);
            const word Xh = (((Eq & pv) + pv) ^ pv) | Eq;
            word Ph = mv | ~(Xh | pv);
            word Mh = pv & Xh;
            const uint32_t bit = w == NW - 1 ? top : (uint32_t)(sizeof(word) * 8 - 1);
            const int hout = (int)((Ph >> bit) & 1) - (int)((Mh >> bit) & 1);
            Ph <<= 1;
            Mh <<= 1;
            if (NW > 1 || HIN != 0) {
                Ph |= (word)(hin > 0);
                Mh |= (word)(hin < 0);
            }
            Pv[w] = Mh | ~(Xv | Ph);
            Mv[w] = Ph & Xv;
            hin = hout;
        }
        score += (uint32_t)hin;
        if (TRACK) {
            if (score < best) {
                best = score;
                cnt = 1;
                first = rel;
            } else if (score == best) {
                cnt++;
            }
        }
    }
};

// ------------------------------------------------------------------------------------------------------------------
// Substitutions only (DESIGN.md section 5.16): H(e) = the mismatches of P against the window S[e-m:e], defined for
// e >= m + the record start.  HamCol keeps one mismatch counter per alignment in flight, bit-sliced: bit j of slice s
// is bit s of the count of the alignment that has met P[0..j].  Per text byte every slice shifts up one bit (a new
// alignment enters at bit 0 with count 0, the one at bit m - 1 leaves), then X = ~PM[c] is added by a ripple carry
// through the slices; the score is bit m - 1 of the slices.  Bits above m - 1 hold partial sums of alignments that
// are already done: they only move up and are never read, so their wrap-around is harmless.  S slices count to BITS
// (6 for one 32-bit word, 7 for one 64-bit word, 8 for the 2-4 word forms, m <= 255).
//
// H(e) depends on S[e-m:e] only, so m - 1 bytes of warm-up before a segment are exact; `fill` counts the bytes a
// column still needs after its reset (at a record start, or at the sequence start) before bit m - 1 holds a whole
// window, and no end is tracked until then.  A column that never tracked an end keeps best = none (~0u), so "has a
// value" is best <= m: unlike Levenshtein there is no end position 0 with score m.
// ------------------------------------------------------------------------------------------------------------------
template <int BITS>
struct HamCol {
    typedef typename NearWord<BITS>::type word;
    static constexpr int NW = near_words(BITS);
    static constexpr int S = BITS == 32 ? 6 : BITS == 64 ? 7 : 8;
    static constexpr uint32_t WB = sizeof(word) * 8;
    word sl[S][NW];
    uint32_t top, fill;
    uint32_t best, cnt, first;
    const word *pm;

    static __device__ __forceinline__ uint32_t none(uint32_t) { return ~0u; }
    static __device__ __forceinline__ bool has(uint32_t best, uint32_t m) { return best <= m; }
    static __device__ __forceinline__ int64_t warm(uint32_t m) { return (int64_t)m - 1; }

    __device__ __forceinline__ void reset(uint32_t m) {
#pragma unroll
        for (int s = 0; s < S; s++)
#pragma unroll
            for (int w = 0; w < NW; w++) sl[s][w] = 0;
        fill = m - 1;
        best = ~0u;
        cnt = 0;
        first = 0;
    }

    template <bool TRACK>
    __device__ __forceinline__ void step(uint32_t c, uint32_t rel) {
#pragma unroll
        for (int s = 0; s < S; s++) {
#pragma unroll
            for (int w = NW - 1; w > 0; w--) sl[s][w] = sl[s][w] << 1 | sl[s][w - 1] >> (WB - 1);
            sl[s][0] <<= 1;
        }
#pragma unroll
        for (int w = 0; w < NW; w++) {
            word carry = ~(NW == 1 ? pm[c * 32] : pm[c * NW + w]);
#pragma unroll
            for (int s = 0; s < S; s++) {
                const word t = sl[s][w] & carry;
                sl[s][w] ^= carry;
                carry = t;
            }
        }
        uint32_t score = 0;
#pragma unroll
        for (int s = 0; s < S; s++) score |= (uint32_t)((sl[s][NW - 1] >> top) & 1) << s;
        if (fill) {
            fill--;
        } else if (TRACK) {
            if (score < best) {
                best = score;
                cnt = 1;
                first = rel;
            } else if (score == best) {
                cnt++;
            }
        }
    }
};

// A column (NearCol or HamCol) over the text bytes [x, end); rel: the end position behind H[x], relative to the
// caller's base
template <bool TRACK, class Col>
__device__ __forceinline__ void near_run(Col &col, const uint8_t *H, int64_t x, int64_t end, uint32_t rel) {
    for (; x < end && (x & 15); x++) col.template step<TRACK>(H[x], rel++);
    for (; x + 16 <= end; x += 16) {
        const uint4 v = __ldg(reinterpret_cast<const uint4 *>(H + x));
        const uint32_t q[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
        for (int j = 0; j < 16; j++) col.template step<TRACK>((q[j >> 2] >> (8 * (j & 3))) & 0xFFu, rel++);
    }
    for (; x < end; x++) col.template step<TRACK>(H[x], rel++);
}

template <class Col, bool REC>
__device__ __forceinline__ void near_scan(NearParams p, RecSet rs) {
    typedef typename Col::word word;
    constexpr int NW = Col::NW;
    extern __shared__ __align__(16) uint64_t near_smem_raw[];
    __shared__ uint32_t s_best[kNearThreads / 32];
    __shared__ uint64_t s_cnt[kNearThreads / 32], s_first[kNearThreads / 32];
    word *pm = reinterpret_cast<word *>(near_smem_raw);
    const uint32_t m = (uint32_t)p.m, lane = threadIdx.x & 31u;

    {  // thread c builds the masks of byte c
        const uint32_t c = threadIdx.x;
        word mask[NW];
#pragma unroll
        for (int w = 0; w < NW; w++) mask[w] = 0;
        for (uint32_t i = 0; i < m; i++)
            if (p.P[i] == c) {
#pragma unroll
                for (int w = 0; w < NW; w++)
                    if ((int)(i / (sizeof(word) * 8)) == w) mask[w] |= (word)1 << (i % (sizeof(word) * 8));
            }
        if (NW == 1) {
            for (int l = 0; l < 32; l++) pm[c * 32 + l] = mask[0];
        } else {
#pragma unroll
            for (int w = 0; w < NW; w++) pm[c * NW + w] = mask[w];
        }
    }
    __syncthreads();

    Col col;
    col.pm = NW == 1 ? pm + lane : pm;
    col.top = (m - 1) % (uint32_t)(sizeof(word) * 8);
    uint32_t tbest = Col::none(m);  // whole sequence: over all tiles of this thread
    uint64_t tcnt = 0, tfirst = kNearNoEnd;

    const int64_t tile = (int64_t)kNearThreads * p.seg;
    for (int64_t base = (int64_t)blockIdx.x * tile; base < p.N; base += (int64_t)gridDim.x * tile) {
        const int64_t a = base + (int64_t)threadIdx.x * p.seg;
        if (a >= p.N) continue;
        const int64_t b = a + p.seg < p.N ? a + p.seg : p.N;
        int64_t lo = 0, hi = p.N;  // the record around the column: [lo, hi), its separator at hi
        uint32_t r = 0;
        if (REC) {
            r = rs.first[a >> kGranuleShift];
            while ((int64_t)rs.off[r + 1] <= a) r++;
            lo = (int64_t)rs.off[r];
            hi = (int64_t)rs.off[r + 1] - 1;
        }
        col.reset(m);
        const int64_t w = a - Col::warm(m) > lo ? a - Col::warm(m) : lo;
        near_run<false>(col, p.H, w, a, 0);
        if (!REC) {
            near_run<true>(col, p.H, a, b, 1);
            near_merge(tbest, tcnt, tfirst, col.best, col.cnt,
                       Col::has(col.best, m) ? (uint64_t)a + col.first : kNearNoEnd);
        } else {
            int64_t x = a;
            for (;;) {
                const int64_t stop = b < hi ? b : hi;
                if (x < stop) near_run<true>(col, p.H, x, stop, (uint32_t)(x + 1 - lo));
                if (Col::has(col.best, m))
                    atomicMin((unsigned long long *)&p.words[r], (unsigned long long)col.best << 32 | col.first);
                if (hi + 1 >= b) break;  // (the record behind the separator starts in another segment, or nowhere)
                r++;
                lo = hi + 1;
                hi = (int64_t)rs.off[r + 1] - 1;
                x = lo;
                col.reset(m);
            }
        }
    }
    if (!REC) {  // the CTA's (minimum, count, first end): warps by shuffle, then thread 0 over the warps
        for (int d = 16; d > 0; d >>= 1) {
            const uint32_t ob = __shfl_down_sync(0xFFFFFFFFu, tbest, d);
            const uint64_t oc = __shfl_down_sync(0xFFFFFFFFu, tcnt, d), of = __shfl_down_sync(0xFFFFFFFFu, tfirst, d);
            near_merge(tbest, tcnt, tfirst, ob, oc, of);
        }
        if (lane == 0) {
            s_best[threadIdx.x >> 5] = tbest;
            s_cnt[threadIdx.x >> 5] = tcnt;
            s_first[threadIdx.x >> 5] = tfirst;
        }
        __syncthreads();
        if (threadIdx.x == 0) {
            for (int i = 1; i < kNearThreads / 32; i++) near_merge(tbest, tcnt, tfirst, s_best[i], s_cnt[i], s_first[i]);
            if (Col::has(tbest, m))
                atomicMin((unsigned long long *)&p.result[0], (unsigned long long)tbest << 48 | tfirst);
            p.partial[2 * blockIdx.x] = tbest;
            p.partial[2 * blockIdx.x + 1] = tcnt;
        }
    }
}

template <int BITS, bool REC>
__global__ void __launch_bounds__(kNearThreads, near_ctas_per_sm(BITS))
k_nearest_scan(NearParams p, RecSet rs) {
    near_scan<NearCol<BITS>, REC>(p, rs);
}

template <int BITS, bool REC>
__global__ void __launch_bounds__(kNearThreads, near_ctas_per_sm(BITS))
k_nearest_hamming_scan(NearParams p, RecSet rs) {
    near_scan<HamCol<BITS>, REC>(p, rs);
}

// n_ends: the ends the CTAs counted at the global minimum, and the end position 0 if that minimum is m_end0 (the
// pattern's length; ~0u under substitutions only, where the end position 0 has no window).  One CTA.
__global__ void k_nearest_count(uint64_t *result, const uint64_t *partial, uint32_t nparts, uint32_t m_end0) {
    const uint64_t best = result[0] >> 48;
    uint64_t sum = threadIdx.x == 0 && best == m_end0 ? 1 : 0;
    for (uint32_t i = threadIdx.x; i < nparts; i += blockDim.x)
        if (partial[2 * i] == best) sum += partial[2 * i + 1];
    if (sum) atomicAdd((unsigned long long *)&result[1], (unsigned long long)sum);
}

// ------------------------------------------------------------------------------------------------------------------
// fzb_nearest_distance_batch / fzb_nearest_best_per_record (DESIGN.md section 5.15): many patterns at once.
//
// k_nearest_batch_scan is the transpose of k_nearest_scan: one lane per pattern, one segment per warp.  The host sorts
// the patterns of one word class (m <= 32 or m <= 64) by length and packs them into groups of 32 lanes; gridDim.y is
// the group.  Every CTA builds its group's table PM[c][lane] (thread c writes byte c's masks of all 32 lanes), so the
// lookup of one text byte by all lanes hits 32 different banks, as in the replicated table of the single scan.  The
// warp walks its segment in lockstep: its text loads and byte extractions are the same for all lanes.  It warms up
// from max(a - 2 max m of its group, record start); a warm-up longer than a lane's own 2 m_i is exact as well (the
// argument at the top of this file: a column started earlier only adds starts that cannot win for e >= w + 2 m_i).
// A lane carries the ORIGINAL ordinal of its pattern (16 bits), so ties are broken by index whatever the grouping;
// idle lanes of a last group (m = 0) run along but never report.
//
// Whole sequence: a lane keeps its minimum and first end over its warp's segments, the CTA combines them per lane in
// shared memory and sends one atomicMin of dist << 48 | first_end per (CTA, pattern) into that pattern's word, which
// the host prefilled with m_i << 48 (the end position 0).
//
// Record sets: at every record end (or segment end) each lane with best < m_i offers key = dist << 48 | ordinal << 32
// | end.  The warp takes the minimum key and, over the lanes whose ordinal differs from the winner's, the minimum pair
// dist << 16 | ordinal; lane 0 sends one atomicMin into best[r] and merges both pairs into top2[r] (best_top2_merge's
// word of best_kernels.cuh).  Both words start as constants: best[r] = (min m_i, its smallest ordinal, end 0) and
// top2[r] = the two smallest pairs (m_i, i).  That is exact although lanes only report scores below their m_i:
// d*_i <= m_i for every pattern, so a pattern left out of the prefill sits behind two patterns j, k whose
// (d*_j, j) <= (m_j, j) < (m_i, i) <= (d*_i, i) -- it can be neither first nor second, and a pattern that is never
// reported has d*_i = m_i with its first end at 0, which is what the prefill says for it.  All updates are minima, so
// the words depend neither on thread, warp or CTA order nor on how records are split over segments.  Under substitutions
// only (k_nearest_hamming_batch_scan, HamCol) nothing has a value before its first window, so both words start empty
// (kBestEmpty) and lanes report every tracked minimum, m_i included.
// ------------------------------------------------------------------------------------------------------------------
constexpr int kNearBatchLanes = 32;
constexpr int kNearBatchMaxM = 64;  // bytes per lane of the pattern buffer

struct NearBatchParams {
    const uint8_t *H;
    int64_t N, seg;         // seg: bytes per warp (a multiple of 16)
    const uint32_t *lanes;  // per lane of every group of this launch: m | ordinal << 16; 0 = idle
    const uint8_t *pats;    // kNearBatchMaxM bytes per lane
    uint64_t *whole;        // per ordinal: dist << 48 | first_end
    uint64_t *best, *top2;  // REC: per record
};

// `pair` (dist << 16 | ordinal) and `pair2` merged into the top2 word of a record (kBestPairNone: nothing)
__device__ __forceinline__ void near_top2_add(uint64_t *top2, uint32_t pair, uint32_t pair2) {
    unsigned long long seen = kBestEmpty;  // (a guess: the first CAS returns the word as it is)
    for (;;) {
        unsigned long long want = best_top2_merge(seen, pair);
        if (pair2 != kBestPairNone) want = best_top2_merge(want, pair2);
        if (want == seen) break;
        const unsigned long long was = atomicCAS((unsigned long long *)top2, seen, want);
        if (was == seen) break;
        seen = was;
    }
}

// The warp's report of one record (all 32 lanes call it with the same record): key as above, ~0 = none
__device__ __forceinline__ void near_batch_report(uint64_t key, uint64_t *best, uint64_t *top2) {
    uint64_t kmin = key;
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) {
        const uint64_t o = __shfl_xor_sync(0xFFFFFFFFu, kmin, d);
        kmin = o < kmin ? o : kmin;
    }
    if (kmin == ~0ull) return;  // (the same for every lane)
    const uint32_t win = (uint32_t)(kmin >> 32);
    uint32_t second = key != ~0ull && ((uint32_t)(key >> 32) & 0xFFFFu) != (win & 0xFFFFu) ? (uint32_t)(key >> 32)
                                                                                          : kBestPairNone;
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) {
        const uint32_t o = __shfl_xor_sync(0xFFFFFFFFu, second, d);
        second = o < second ? o : second;
    }
    if ((threadIdx.x & 31u) == 0) {
        atomicMin((unsigned long long *)best, (unsigned long long)kmin);
        near_top2_add(top2, win, second);
    }
}

template <class Col, bool REC>
__device__ __forceinline__ void near_batch_scan(NearBatchParams p, RecSet rs) {
    static_assert(Col::NW == 1, "one word per lane");
    typedef typename Col::word word;
    extern __shared__ __align__(16) uint64_t near_smem_raw[];
    __shared__ __align__(16) uint8_t s_pat[kNearBatchLanes * kNearBatchMaxM];
    __shared__ uint32_t s_m[kNearBatchLanes];
    __shared__ uint64_t s_key[kNearThreads / 32][kNearBatchLanes];
    word *pm = reinterpret_cast<word *>(near_smem_raw);
    const uint32_t lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
    const uint32_t *lanes = p.lanes + (size_t)blockIdx.y * kNearBatchLanes;
    const uint8_t *pats = p.pats + (size_t)blockIdx.y * kNearBatchLanes * kNearBatchMaxM;

    for (uint32_t i = threadIdx.x; i < kNearBatchLanes * kNearBatchMaxM; i += kNearThreads) s_pat[i] = pats[i];
    if (threadIdx.x < kNearBatchLanes) s_m[threadIdx.x] = lanes[threadIdx.x] & 0xFFFFu;
    __syncthreads();
    {  // thread c builds the masks of byte c for every lane
        const uint32_t c = threadIdx.x;
        for (int l = 0; l < kNearBatchLanes; l++) {
            word mask = 0;
            for (uint32_t i = 0; i < s_m[l]; i++)
                if (s_pat[l * kNearBatchMaxM + i] == c) mask |= (word)1 << i;
            pm[c * kNearBatchLanes + l] = mask;
        }
    }
    __syncthreads();

    const uint32_t info = lanes[lane], ord = info >> 16;
    const bool idle = (info & 0xFFFFu) == 0;
    const uint32_t m = idle ? 1u : info & 0xFFFFu;
    uint32_t gm = m;  // the longest pattern of the group: the warm-up of every lane
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) {
        const uint32_t o = __shfl_xor_sync(0xFFFFFFFFu, gm, d);
        gm = o > gm ? o : gm;
    }
    Col col;
    col.pm = pm + lane;
    col.top = m - 1;
    uint32_t tbest = Col::none(m);  // whole sequence: over all segments of this warp
    uint64_t tfirst = kNearNoEnd;

    const int64_t tile = (int64_t)(kNearThreads / 32) * p.seg;
    for (int64_t base = (int64_t)blockIdx.x * tile; base < p.N; base += (int64_t)gridDim.x * tile) {
        const int64_t a = base + (int64_t)warp * p.seg;
        if (a >= p.N) continue;
        const int64_t b = a + p.seg < p.N ? a + p.seg : p.N;
        int64_t lo = 0, hi = p.N;  // the record around the column: [lo, hi), its separator at hi
        uint32_t r = 0;
        if (REC) {
            r = rs.first[a >> kGranuleShift];
            while ((int64_t)rs.off[r + 1] <= a) r++;
            lo = (int64_t)rs.off[r];
            hi = (int64_t)rs.off[r + 1] - 1;
        }
        col.reset(m);
        const int64_t w = a - Col::warm(gm) > lo ? a - Col::warm(gm) : lo;
        near_run<false>(col, p.H, w, a, 0);
        if (!REC) {
            near_run<true>(col, p.H, a, b, 1);
            if (col.best < tbest) {  // (segments come in increasing order: an equal minimum keeps the earlier end)
                tbest = col.best;
                tfirst = (uint64_t)a + col.first;
            }
        } else {
            int64_t x = a;
            for (;;) {
                const int64_t stop = b < hi ? b : hi;
                if (x < stop) near_run<true>(col, p.H, x, stop, (uint32_t)(x + 1 - lo));
                const uint64_t key = !idle && Col::has(col.best, m)
                                         ? (uint64_t)col.best << 48 | (uint64_t)ord << 32 | col.first
                                         : ~0ull;
                near_batch_report(key, p.best + r, p.top2 + r);
                if (hi + 1 >= b) break;  // (the record behind the separator starts in another segment, or nowhere)
                r++;
                lo = hi + 1;
                hi = (int64_t)rs.off[r + 1] - 1;
                x = lo;
                col.reset(m);
            }
        }
    }
    if (!REC) {  // per lane over the warps of the CTA, then one atomicMin per (CTA, pattern)
        s_key[warp][lane] = !idle && Col::has(tbest, m) ? (uint64_t)tbest << 48 | tfirst : ~0ull;
        __syncthreads();
        if (warp == 0) {
            uint64_t key = s_key[0][lane];
            for (int i = 1; i < kNearThreads / 32; i++) key = s_key[i][lane] < key ? s_key[i][lane] : key;
            if (key != ~0ull) atomicMin((unsigned long long *)&p.whole[ord], (unsigned long long)key);
        }
    }
}

template <int BITS, bool REC>
__global__ void __launch_bounds__(kNearThreads, near_ctas_per_sm(BITS))
k_nearest_batch_scan(NearBatchParams p, RecSet rs) {
    near_batch_scan<NearCol<BITS>, REC>(p, rs);
}

template <int BITS, bool REC>
__global__ void __launch_bounds__(kNearThreads, near_ctas_per_sm(BITS))
k_nearest_hamming_batch_scan(NearBatchParams p, RecSet rs) {
    near_batch_scan<HamCol<BITS>, REC>(p, rs);
}

// A pattern of 65-255 symbols scanned alone by k_nearest_scan<BITS, true> (k_nearest_hamming_scan): its per-record
// words (dist << 32 | end) below `lim` folded into best / top2 as the lanes of the batch scan report.  lim is m for
// Levenshtein (the prefill stands for d = m) and m + 1 under substitutions only (d = m is reported, and the empty
// word, dist 0xFFFFFFFF, is not).  One thread per record.
__global__ void k_nearest_fold(const uint64_t *words, uint64_t nrec, uint32_t lim, uint32_t ord, uint64_t *best,
                               uint64_t *top2) {
    const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
    for (uint64_t r = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; r < nrec; r += stride) {
        const uint64_t w = words[r];
        const uint32_t d = (uint32_t)(w >> 32);
        if (d >= lim) continue;
        atomicMin((unsigned long long *)&best[r], (unsigned long long)d << 48 | (uint64_t)ord << 32 | (w & 0xFFFFFFFFull));
        near_top2_add(&top2[r], d << 16 | ord, kBestPairNone);
    }
}

// ------------------------------------------------------------------------------------------------------------------
// Anchored nearest matches (DESIGN.md section 5.18): fzb_nearest_per_record / fzb_nearest_best_per_record with
// FZB_F_ANCHOR_START or FZB_F_ANCHOR_END.  For the pattern P (m symbols) and a record R (n symbols):
//   'start'  A(e) = lev(P, R[0:e]), e in 0..n: dist = min A, pos = the smallest e that reaches it;
//   'end'    B(s) = lev(P, R[s:n]): the same problem on (P reversed, R reversed), so the kernel walks the record
//            backwards with the reversed pattern's table (the host reverses it) and pos = n - s, the end in the
//            mirrored record -- the smallest such pos is the largest s.  k_nearest_anchored_flip turns pos into s.
// A is the bottom row of the prefix-anchored table (D[0][j] = j: NearCol::step with HIN = +1).  A(0) = m and
// A(e) >= e - m, so no e >= m + best can win: a lane reads at most min(n, 2m) symbols and stops at e - m >= best.
// Under substitutions only (HAM) dist = the mismatches of P against R[0:m] ('start', pos = m) or R[n-m:n] ('end',
// pos = m as well, the mirror's end); a record shorter than m has no value.  Either way a window never leaves its
// record, so a separator is never read.
//
// Layout: one record per lane group of g lanes (g a power of two, 1 to 32), lane l on pattern slot l % g of the
// CTA row's group (blockIdx.y), records grid-stride.  The table is k_nearest_batch_scan's PM[c][lane], lane l
// holding the masks of its own slot, so 32 lanes never share a bank.  BATCH: every lane group sends the smallest
// key dist << 48 | ordinal << 32 | pos and the runner-up pair of near_batch_report into best[r] / top2[r], over the
// prefills of section 5.15 / 5.16 (a Levenshtein lane reports only dist < m: the prefill (m_i, i, pos 0) is A(0)).
// Single pattern (!BATCH): g = 1, one lane per record writes words[r] = dist << 32 | pos (all ones: no value),
// without prefill; with 2-4 words (m <= 255) the table is [c][word], shared by all lanes, as in k_nearest_scan.
// `steps` counts the symbols read: per lane group, the longest window one of its lanes read.
// ------------------------------------------------------------------------------------------------------------------
struct NearAnchParams {
    const uint8_t *H;
    uint64_t nrec;
    const uint32_t *lanes;  // BATCH: m | ordinal << 16 per lane of every group (0 = idle), as NearBatchParams
    const uint8_t *pats;    // BATCH: kNearBatchMaxM bytes per lane
    uint64_t *words;        // single: dist << 32 | pos per record
    uint64_t *best, *top2;  // BATCH: per record
    uint64_t *steps;        // the symbols read (added to)
    int32_t m, g, end;      // m: single; g: lanes per record; end: 'end' (walk the records backwards)
    uint8_t P[256];         // single
};

template <int BITS, bool HAM, bool BATCH>
__global__ void __launch_bounds__(kNearThreads, near_ctas_per_sm(BITS))
k_nearest_anchored(NearAnchParams p, RecSet rs) {
    typedef typename NearWord<BITS>::type word;
    constexpr int NW = near_words(BITS);
    constexpr uint32_t WB = sizeof(word) * 8;
    static_assert(!BATCH || NW == 1, "one word per lane");
    extern __shared__ __align__(16) uint64_t near_smem_raw[];
    __shared__ __align__(16) uint8_t s_pat[BATCH ? kNearBatchLanes * kNearBatchMaxM : 256];
    __shared__ uint32_t s_m[kNearBatchLanes];
    word *pm = reinterpret_cast<word *>(near_smem_raw);
    const uint32_t lane = threadIdx.x & 31u, g = BATCH ? (uint32_t)p.g : 1u, slot = lane % g;

    if (BATCH) {
        const uint8_t *pats = p.pats + (size_t)blockIdx.y * kNearBatchLanes * kNearBatchMaxM;
        for (uint32_t i = threadIdx.x; i < kNearBatchLanes * kNearBatchMaxM; i += kNearThreads) s_pat[i] = pats[i];
        if (threadIdx.x < kNearBatchLanes) s_m[threadIdx.x] = p.lanes[blockIdx.y * kNearBatchLanes + threadIdx.x] & 0xFFFFu;
    } else {
        s_pat[threadIdx.x] = p.P[threadIdx.x];
    }
    __syncthreads();
    {  // thread c builds the masks of byte c: per lane (of its slot) with one word, [c][word] with more
        const uint32_t c = threadIdx.x;
        if (NW == 1) {
            for (uint32_t l = 0; l < 32; l++) {
                const uint32_t k = BATCH ? l % g : 0, mk = BATCH ? s_m[k] : (uint32_t)p.m;
                word mask = 0;
                for (uint32_t i = 0; i < mk; i++)
                    if (s_pat[(BATCH ? k * kNearBatchMaxM : 0) + i] == c) mask |= (word)1 << i;
                pm[c * 32 + l] = mask;
            }
        } else {
            word mask[NW];
#pragma unroll
            for (int w = 0; w < NW; w++) mask[w] = 0;
            for (uint32_t i = 0; i < (uint32_t)p.m; i++)
                if (s_pat[i] == c) {
#pragma unroll
                    for (int w = 0; w < NW; w++)
                        if ((int)(i / WB) == w) mask[w] |= (word)1 << (i % WB);
                }
#pragma unroll
            for (int w = 0; w < NW; w++) pm[c * NW + w] = mask[w];
        }
    }
    __syncthreads();

    const uint32_t info = BATCH ? p.lanes[blockIdx.y * kNearBatchLanes + slot] : (uint32_t)p.m;
    const uint32_t m = info & 0xFFFFu, ord = info >> 16;  // (m = 0: an idle lane)
    const word *tab = NW == 1 ? pm + lane : pm;
    auto mask_of = [&](uint32_t c, int w) -> word { return NW == 1 ? tab[c * 32] : tab[c * NW + w]; };
    NearCol<BITS> col;
    col.pm = tab;
    col.top = (m - 1) % WB;
    uint64_t nread = 0;  // lane group leaders: the symbols their group read

    const uint64_t per = (uint64_t)(kNearThreads / 32) * (32 / g);  // records per CTA and round
    // (the trip count is the same for the lanes of a warp: the collectives below take all 32)
    for (uint64_t base = (uint64_t)blockIdx.x * per + (threadIdx.x >> 5) * (32 / g); base < p.nrec;
         base += (uint64_t)gridDim.x * per) {
        const uint64_t r = base + lane / g;
        uint32_t dist = ~0u, pos = 0, read = 0;
        if (r < p.nrec && m) {
            const int64_t lo = (int64_t)rs.off[r], hi = (int64_t)rs.off[r + 1] - 1;
            const uint32_t n = (uint32_t)(hi - lo);
            if (HAM) {
                if (n >= m) {
                    const int64_t at = p.end ? hi - m : lo;
                    word hit[NW];
#pragma unroll
                    for (int w = 0; w < NW; w++) hit[w] = 0;
                    for (uint32_t i = 0; i < m; i++) {
                        const uint32_t c = __ldg(p.H + at + i);
#pragma unroll
                        for (int w = 0; w < NW; w++)
                            if ((int)(i / WB) == w) hit[w] |= mask_of(c, w) & (word)1 << (i % WB);
                    }
                    uint32_t same = 0;
#pragma unroll
                    for (int w = 0; w < NW; w++) same += WB == 64 ? __popcll((uint64_t)hit[w]) : __popc((uint32_t)hit[w]);
                    dist = m - same;
                    pos = read = m;
                }
            } else {
#pragma unroll
                for (int w = 0; w < NW; w++) {
                    col.Pv[w] = ~(word)0;
                    col.Mv[w] = 0;
                }
                col.score = dist = m;
                const uint32_t lim = n < 2 * m ? n : 2 * m;
                for (uint32_t e = 1; e <= lim && (int)e - (int)m < (int)dist; e++) {
                    col.template step<false, 1>(__ldg(p.H + (p.end ? hi - e : lo + e - 1)), 0);
                    read = e;
                    if (col.score < dist) {
                        dist = col.score;
                        pos = e;
                    }
                }
            }
        }
        if (!BATCH) {
            if (r < p.nrec) p.words[r] = dist == ~0u ? kBestEmpty : (uint64_t)dist << 32 | pos;
            nread += read;
            continue;
        }
        // the lane group's smallest key and, over its other patterns, the smallest pair (near_batch_report per group)
        const bool has = dist != ~0u && (HAM || dist < m);
        const uint64_t key = has ? (uint64_t)dist << 48 | (uint64_t)ord << 32 | pos : ~0ull;
        uint64_t kmin = key;
        for (uint32_t d = g >> 1; d; d >>= 1) {
            const uint64_t o = __shfl_xor_sync(0xFFFFFFFFu, kmin, d);
            kmin = o < kmin ? o : kmin;
        }
        const uint32_t win = (uint32_t)(kmin >> 32);
        uint32_t second = has && ord != (win & 0xFFFFu) ? (uint32_t)(key >> 32) : kBestPairNone;
        for (uint32_t d = g >> 1; d; d >>= 1) {
            const uint32_t o = __shfl_xor_sync(0xFFFFFFFFu, second, d);
            second = o < second ? o : second;
            const uint32_t oread = __shfl_xor_sync(0xFFFFFFFFu, read, d);
            read = oread > read ? oread : read;
        }
        if (slot == 0 && r < p.nrec) {
            nread += read;
            if (kmin != ~0ull) {
                atomicMin((unsigned long long *)&p.best[r], (unsigned long long)kmin);
                near_top2_add(&p.top2[r], win, second);
            }
        }
    }
    for (int d = 16; d > 0; d >>= 1) nread += __shfl_xor_sync(0xFFFFFFFFu, nread, d);
    if (lane == 0 && nread) atomicAdd((unsigned long long *)p.steps, (unsigned long long)nread);
}

// 'end': the pos of every word with a value (dist << 32 | pos, or a best key) from the mirrored record's end to the
// start in the record, n - pos.  One thread per record.
__global__ void k_nearest_anchored_flip(uint64_t *words, uint64_t nrec, RecSet rs) {
    const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
    for (uint64_t r = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; r < nrec; r += stride) {
        const uint64_t w = words[r];
        if (w == kBestEmpty) continue;
        const uint64_t n = rs.off[r + 1] - 1 - rs.off[r];
        words[r] = (w & ~0xFFFFFFFFull) | (n - (w & 0xFFFFFFFFull));
    }
}

}  // namespace fzb
