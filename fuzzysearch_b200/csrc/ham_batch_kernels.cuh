// ham_batch_kernels.cuh -- many substitutions-only (Hamming) patterns over one haystack in ONE pass.
//
// Filter (pigeonhole, exact for substitutions): cut pattern P (m symbols, at most k substitutions) into k+1 pieces
// of L = floor(m/(k+1)) symbols at offsets o_j = j*L.  An occurrence at start p has at least one piece that matches
// exactly at g = p + o_j, and with no insertions or deletions the candidate start is exactly g - o_j: no granules,
// no windows, no de-duplication set.
//   k_ham_batch_scan  streams the haystack once.  At EVERY position g a key built from the symbols at g is tested
//        against a shared-memory table holding the keys of all pieces of all patterns of the pass; on a hit the lane
//        walks the L2-resident posting list (pattern, piece j) of that key, and for each posting counts the
//        mismatches of P against H[g-o_j : g-o_j+m] (stopping once they pass k).  It emits (p, p+m, d) -- tagged with
//        the pattern's ordinal, ngram = pid << 8 -- only if d <= k, piece j itself matches exactly and no piece i < j
//        does: each (pattern, start) is emitted exactly once, by its first exact piece.
//   Two key widths (the host picks one from the haystack's byte statistics):
//     text  (TWO_BIT = false): the first min(L, 4) bytes at g -- one width per pass, 4 or 3 (key_mask) -- hashed into
//           a 2^20-bit table (128 KiB); a hit must also pass a second-level 2^23-bit table in L2 (independent hash)
//           before the lane probes the postings.
//     DNA   (TWO_BIT = true):  the 2-bit codes of the 8 symbols at g (a 256-entry byte -> code table built from the
//           pass's pattern bytes), an exact 64 Ki-bit table (8 KiB).  A piece of L < 8 symbols is entered under
//           every completion of its key.  Bytes outside the pattern alphabet alias to some code; that only adds
//           candidates, because the verification compares bytes.
#pragma once
#include "batch_kernels.cuh"

namespace fzb {

struct HamBatchParams {
    MultiParams mp;       // H, geometry, key table (bits; text: bits2 too), gtab keyed by the key, postings
                          // pid << 8 | piece, pinfo m | k << 8 | L << 16, counters (CNT_CAND = candidates verified)
    const BatchPat *pats;
    RawRec *out;
    uint32_t cap;
    uint32_t key_mask;    // text keys: 0xFFFFFFFF (4 bytes) or 0x00FFFFFF (3 bytes)
    uint8_t code[256];    // 2-bit keys: byte -> code
};

// 4 bytes -> 4 bits: bit i set iff byte i of x is non-zero
__device__ __forceinline__ uint32_t hb_nonzero_nibble(uint32_t x) {
    const uint32_t nz = (((x & 0x7F7F7F7Fu) + 0x7F7F7F7Fu) | x) & 0x80808080u;
    return (((nz >> 7) * 0x00204081u) >> 21) & 0xFu;
}

// Position g (global) carries `key`: walk its postings, verify each candidate start; -> candidates verified.
// REC: `rs` is the record set (one argument, by value); a start is emitted only if its occurrence lies inside one record.  Without
// records the pack is empty, so the call passes exactly the arguments it passed before record sets existed.
template <bool REC, class... Rec>
__device__ __noinline__ uint32_t hb_confirm(const HamBatchParams &p, uint32_t key, int64_t g, Rec... rs) {
    uint32_t n = 0;
    uint32_t slot = (key * kGramMul) & p.mp.gtab_mask;
    for (;;) {
        const uint2 e = __ldg(p.mp.gtab + slot);
        if (e.y == 0u) return n;
        if (e.x == key) {
            const uint32_t first = e.y & 0xFFFFFFu, cnt = e.y >> 24;
            for (uint32_t i = 0; i < cnt; i++) {
                const uint32_t post = __ldg(p.mp.postings + first + i);
                const uint32_t pid = post >> 8;
                const int j = (int)(post & 0xFFu);
                const uint32_t info = __ldg(p.mp.pinfo + pid);
                const int m = (int)(info & 0xFFu), k = (int)((info >> 8) & 0xFFu), L = (int)((info >> 16) & 0xFFu);
                const int64_t st = g - (int64_t)j * L;
                if (st < p.mp.own_lo || st >= p.mp.own_hi || st + m > p.mp.N) continue;
                n++;
                // mismatch mask of P against H[st : st+m], four bytes at a time (the buffer is padded behind its end)
                const int64_t off = st - p.mp.buf_lo;
                const uint32_t *T = reinterpret_cast<const uint32_t *>(p.mp.H + (off & ~(int64_t)3));
                const uint32_t sh = 8u * (uint32_t)(off & 3);
                const uint32_t *Pw = reinterpret_cast<const uint32_t *>(p.pats[pid].P);
                unsigned long long mm = 0ull;
                int nd = 0;
                uint32_t lo = __ldg(T);
                for (int w = 0; 4 * w < m; w++) {
                    const uint32_t hi = __ldg(T + w + 1);
                    uint32_t bits = hb_nonzero_nibble(__funnelshift_r(lo, hi, sh) ^ __ldg(Pw + w));
                    lo = hi;
                    if (4 * w + 4 > m) bits &= (1u << (m - 4 * w)) - 1u;
                    mm |= (unsigned long long)bits << (4 * w);
                    nd += __popc(bits);
                    if (nd > k) break;
                }
                if (nd > k) continue;
                const unsigned long long piece = L >= 64 ? ~0ull : (1ull << L) - 1ull;
                if (mm & (piece << (j * L))) continue;  // the key matched, the piece does not (hash / code aliasing)
                bool first_exact = true;
                for (int q = 0; q < j; q++)
                    if (!(mm & (piece << (q * L)))) first_exact = false;  // an earlier piece emits this start
                if constexpr (REC)
                    if (first_exact) first_exact = ham_in_record<true>(rs..., st, m);
                if (first_exact) emit(p.out, p.cap, p.mp.counters, st, st + m, st, nd, (int)(pid << 8), false);
            }
        }
        slot = (slot + 1) & p.mp.gtab_mask;
    }
}

template <bool TWO_BIT, bool REC>
__global__ void __launch_bounds__(kMultiThreads, 1)
k_ham_batch_scan(const __grid_constant__ HamBatchParams p, int64_t nvec, int64_t ntiles, const RecSet rs) {
    extern __shared__ __align__(16) uint32_t hb_tbl[];
    __shared__ uint8_t sCode[256];
    constexpr int kWords = TWO_BIT ? kHbKeyWords : kMultiTblWords;
    for (int i = threadIdx.x; i < kWords / 4; i += kMultiThreads)
        reinterpret_cast<uint4 *>(hb_tbl)[i] = __ldg(reinterpret_cast<const uint4 *>(p.mp.bits) + i);
    for (int i = threadIdx.x; i < 256; i += kMultiThreads) sCode[i] = p.code[i];
    __syncthreads();
    const int lane = threadIdx.x & 31;
    const uint4 *base = reinterpret_cast<const uint4 *>(p.mp.H);
    uint32_t cand = 0;
    for (int64_t t = blockIdx.x; t < ntiles; t += gridDim.x) {
#pragma unroll 1
        for (int u = 0; u < kMultiUnroll; u++) {
            const int64_t v = t * kMultiTileVecs + (int64_t)u * kMultiThreads + threadIdx.x;
            const uint4 d = (v < nvec) ? ldg_stream(base + v) : make_uint4(0, 0, 0, 0);
            uint32_t nx = __shfl_down_sync(0xFFFFFFFFu, d.x, 1);  // the 8 bytes after my 16
            uint32_t ny = __shfl_down_sync(0xFFFFFFFFu, d.y, 1);
            if (lane == 31 && v < nvec) {  // padded buffer
                const uint2 e = __ldg(reinterpret_cast<const uint2 *>(base + v + 1));
                nx = e.x;
                ny = e.y;
            }
            const uint32_t ws[6] = {d.x, d.y, d.z, d.w, nx, ny};
            uint32_t acc = 0;  // bit (15 - b) <-> position b of my vector
            unsigned long long codes = 0ull;  // 2-bit codes of my 16 bytes and the 7 after them
            if (TWO_BIT) codes = key_codes(sCode, ws);
#pragma unroll
            for (int b = 0; b < 16; b++) {
                uint32_t h;
                if (TWO_BIT)
                    h = (uint32_t)(codes >> (2 * b)) & 0xFFFFu;
                else
                    h = multi_hash(__funnelshift_r(ws[b >> 2], ws[(b >> 2) + 1], 8 * (b & 3)) & p.key_mask);
                acc = acc * 2u + ((hb_tbl[h >> 5] >> (h & 31u)) & 1u);
            }
            const int64_t off = v * 16;
            while (acc) {
                const int bit = 31 - __clz(acc);
                acc &= ~(1u << bit);
                const int b = 15 - bit;
                if (off + b >= p.mp.buf_len) continue;
                const uint32_t key = TWO_BIT ? (uint32_t)(codes >> (2 * b)) & 0xFFFFu
                                             : __funnelshift_r(ws[b >> 2], ws[(b >> 2) + 1], 8 * (b & 3)) & p.key_mask;
                if (!TWO_BIT) {  // second level (L2): most false positives of the hashed table stop here
                    const uint32_t h2 = multi_hash2(key);
                    if (!((__ldg(p.mp.bits2 + (h2 >> 5)) >> (h2 & 31u)) & 1u)) continue;
                }
                if constexpr (REC)
                    cand += hb_confirm<true>(p, key, p.mp.buf_lo + off + b, rs);
                else
                    cand += hb_confirm<false>(p, key, p.mp.buf_lo + off + b);
            }
        }
    }
#pragma unroll
    for (int s = 16; s > 0; s >>= 1) cand += __shfl_down_sync(0xFFFFFFFFu, cand, s);
    if (lane == 0 && cand) atomicAdd(&p.mp.counters[CNT_CAND], cand);
}

}  // namespace fzb
