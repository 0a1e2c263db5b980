// align_kernels.cuh -- fzb_align (DESIGN.md section 5.17): the edit operations of one pattern against one window of the
// resident sequence, one warp per item.
//
// An item is (pattern P of m symbols, window [s, e) in buffer coordinates, cost bound d).  Its class decides the cost
// model: exact and substitutions-only items compare the m symbols of the window position by position; Levenshtein
// items take the unit-cost edit distance; generic items the smallest X + I + D with X <= S', I <= I', D <= D' and a
// total <= L'.  The host prepares every item (clamped bounds, record clipping, shared-memory need) and sorts the items
// into launches by their shared-memory need; one CTA of one warp runs one item at a time.
//
// The dynamic-programming items sweep the anti-diagonals a = i + j of their table across the warp's lanes (a cell
// (i, j) needs (i-1, j-1) on a - 2 and (i-1, j), (i, j-1) on a - 1).  Only a band of diagonals k = j - i is swept:
//   Levenshtein: a cell on an alignment of cost <= d has |k| + |w - m - k| <= d, so k lies within (d - |w - m|) / 2 of
//                the diagonals between 0 and w - m; with |w - m| > d there is no alignment.
//   generic:     one layer per number l of insertions used, 0 <= l <= I'; on layer l the deletions used are l - k, so
//                the layer holds the D' + 1 diagonals l - D' .. l, and a cell holds the fewest substitutions of a path
//                that reaches it with l insertions and l - k deletions.
// Inside the band the banded table equals the full one on every cell of an optimal path (every such cell is reached
// by an optimal prefix that stays in the band), so the traceback below is the full table's.  Three rings of int16
// values hold the last three anti-diagonals; each cell also stores a 2-bit traceback code in shared memory: 0 the
// diagonal step (= or X), 1 a deletion (a pattern symbol missing from the sequence, from (i-1, j)), 2 an insertion (a
// sequence symbol with no counterpart in the pattern, from (i, j-1), on generic layer l - 1), the first of them, in
// that order, that reaches the cell's value.  Lane 0 then walks the codes back from (m, w): the canonical alignment
// prefers the diagonal, then a deletion, then an insertion at every step.
//
// A free-start Levenshtein item first sweeps the reversed pattern against the reversed sequence from e down to the
// record's first symbol (band |k| <= d, values only, row m kept): row m at column j is lev(P, S[e-j : e)), and the
// largest j where it equals d gives the smallest start.  Then the anchored sweep runs on [s, e).
#pragma once
#include "common.cuh"

namespace fzb {

constexpr int kAlignSmemMax = 64 * 1024;  // dynamic shared memory of one item at most (FZB_E_UNSUPPORTED above)
constexpr int kAlignInf = 0x3FFF;
constexpr int kAlignBuckets = 4;  // launches by shared-memory need: <= 2, 8, 24 KiB, kAlignSmemMax
constexpr int kAlignBucketBytes[kAlignBuckets] = {2 * 1024, 8 * 1024, 24 * 1024, kAlignSmemMax};
enum : uint8_t { kAlignExact = 0, kAlignHamming = 1, kAlignLevenshtein = 2, kAlignGeneric = 3 };

struct AlignItem {
    int64_t s;        // window start (buffer coordinates); -1: free start (Levenshtein only)
    int64_t e;        // window end
    int64_t lo;       // the first symbol of the record holding the window (0 without a record set)
    uint64_t op_off;  // where the item's ops go
    uint64_t idx;     // the item's index in the caller's arrays
    uint32_t pat_off; // the pattern in the pattern blob
    int32_t d;        // the cost bound, clamped (see prepare_align_item in api.cu)
    uint16_t m;
    uint8_t cls;
    uint8_t pad_;
    uint16_t subs, ins, dels, lim;  // generic: S', I', D', L' (each clamped to d)
};

// The bytes one sweep needs: three int16 rings of layers x (bw / 2 + 2) values (an anti-diagonal holds at most
// bw / 2 + 1 cells of a layer), then `extra` bytes at a 16-byte boundary.
__host__ __device__ __forceinline__ uint32_t align_ring(int bw) { return (uint32_t)(bw / 2 + 2); }
__host__ __device__ __forceinline__ uint64_t align_vals_bytes(int layers, int bw) {
    return ((uint64_t)6 * layers * align_ring(bw) + 15) & ~15ull;
}
// the 2-bit traceback codes of layers x (m + 1) rows x bw diagonals
__host__ __device__ __forceinline__ uint64_t align_table_bytes(int layers, int m, int bw) {
    return 4 * (((uint64_t)layers * (m + 1) * bw + 15) / 16);
}
// Levenshtein band of an anchored window: [kmin, kmin + bw); bw == 0 when |w - m| > d (no alignment)
__host__ __device__ __forceinline__ int align_lev_band(int m, int64_t w, int d, int *kmin) {
    const int64_t delta = w - m, ad = delta < 0 ? -delta : delta;
    if (ad > d) return 0;
    const int h = (int)((d - ad) / 2);
    *kmin = (int)(delta < 0 ? delta : 0) - h;
    return (int)ad + 2 * h + 1;
}

struct AlignSweep {
    const uint8_t *P;  // the pattern
    const uint8_t *T;  // forward: the window's first symbol; reversed: the symbol after the window's last
    int m, w;
    bool rev;          // reversed: row i reads P[m - i], column j reads T[-j]
    bool generic;
    int layers, bw, klo0;  // layer l holds the diagonals klo0 + (generic ? l : 0) .. + bw - 1
    int S, L;              // generic: X <= S, total <= L
    int16_t *vals;         // 3 rings of layers x align_ring(bw)
    uint32_t *table;       // traceback codes, or null
    int16_t *rowm;         // row m by diagonal - klo0, or null
};

__device__ __forceinline__ int align_floor2(int x) { return x >> 1; }  // (arithmetic shift: floor for negatives)

__device__ void align_sweep(const AlignSweep &g, int lane) {
    const int R = (int)align_ring(g.bw), cmax = g.bw / 2 + 1, per = g.layers * cmax;
    for (int a = 0; a <= g.m + g.w; a++) {
        int16_t *cur = g.vals + (a % 3) * g.layers * R;
        const int16_t *p1 = g.vals + ((a + 2) % 3) * g.layers * R, *p2 = g.vals + ((a + 1) % 3) * g.layers * R;
        for (int t = lane; t < per; t += 32) {
            const int l = t / cmax;
            const int klo = g.klo0 + (g.generic ? l : 0), khi = klo + g.bw - 1;
            int ilo = max(max(0, a - g.w), -align_floor2(khi - a));  // ceil((a - khi) / 2)
            const int ihi = min(min(g.m, a), align_floor2(a - klo));
            const int i = ilo + t % cmax;
            if (i > ihi) continue;
            const int j = a - i, k = j - i;
            int best, code = 0;
            if (i == 0 && j == 0) {
                best = l == 0 ? 0 : kAlignInf;
            } else {
                int vd = kAlignInf, vu = kAlignInf, vl = kAlignInf;
                if (i > 0 && j > 0) {
                    const uint8_t pc = g.rev ? g.P[g.m - i] : g.P[i - 1];
                    const uint8_t tc = g.rev ? g.T[-j] : g.T[j - 1];
                    vd = p2[l * R + (i - 1) % R] + (pc != tc);
                }
                if (i > 0 && k + 1 <= khi) vu = p1[l * R + (i - 1) % R] + (g.generic ? 0 : 1);
                const int ll = g.generic ? l - 1 : l;
                if (j > 0 && ll >= 0 && k - 1 >= g.klo0 + (g.generic ? ll : 0))
                    vl = p1[ll * R + i % R] + (g.generic ? 0 : 1);
                best = min(vd, min(vu, vl));
                code = best == vd ? 0 : best == vu ? 1 : 2;
                if (best >= kAlignInf || (g.generic && (best > g.S || best + l + (l - k) > g.L))) best = kAlignInf;
            }
            cur[l * R + i % R] = (int16_t)best;
            if (g.table) {
                const uint64_t cell = ((uint64_t)l * (g.m + 1) + i) * g.bw + (k - klo);
                atomicOr(&g.table[cell >> 4], (uint32_t)code << (2 * (cell & 15)));
            }
            if (g.rowm && i == g.m) g.rowm[k - g.klo0] = (int16_t)best;
        }
        __syncwarp();
    }
}

struct AlignOut {
    int64_t *start;
    int32_t *cost, *n_subs, *n_ins, *n_dels;
    uint8_t *ops;
};

__device__ __forceinline__ void align_put(const AlignOut &o, uint64_t idx, int64_t s, int c, int x, int ins, int del) {
    o.start[idx] = s;
    o.cost[idx] = c;
    o.n_subs[idx] = x;
    o.n_ins[idx] = ins;
    o.n_dels[idx] = del;
}

// One warp (the whole CTA) per item, items[0 .. n) of one launch; `smem` bytes of dynamic shared memory each.
__global__ void __launch_bounds__(32) k_align(const uint8_t *H, const uint8_t *patterns, const AlignItem *items,
                                              uint64_t n, AlignOut out) {
    extern __shared__ __align__(16) uint8_t al_smem[];
    const int lane = threadIdx.x;
    for (uint64_t it = blockIdx.x; it < n; it += gridDim.x) {
        const AlignItem item = items[it];
        const uint8_t *P = patterns + item.pat_off;
        const int m = item.m, d = item.d;
        int64_t s = item.s;
        if (item.cls == kAlignExact || item.cls == kAlignHamming) {  // no gaps: m position-by-position comparisons
            if (s < 0) s = item.e - m;
            if (s < item.lo) {
                if (lane == 0) align_put(out, item.idx, -1, -1, -1, -1, -1);
                continue;
            }
            int x = 0;
            for (int j0 = 0; j0 < m; j0 += 32) {
                const bool ne = j0 + lane < m && P[j0 + lane] != H[s + j0 + lane];
                x += __popc(__ballot_sync(0xFFFFFFFFu, ne));
            }
            if (x > d) {
                if (lane == 0) align_put(out, item.idx, -1, -1, -1, -1, -1);
                continue;
            }
            for (int j = lane; j < m; j += 32) out.ops[item.op_off + j] = P[j] != H[s + j] ? 'X' : '=';
            if (lane == 0) align_put(out, item.idx, s, x, x, 0, 0);
            continue;
        }
        const bool generic = item.cls == kAlignGeneric;
        if (s < 0) {  // free start: the reversed sweep from e over at most m + d symbols of the record
            const int64_t lo = item.e - m - d > item.lo ? item.e - m - d : item.lo;
            AlignSweep r{};
            r.P = P;
            r.T = H + item.e;
            r.m = m;
            r.w = (int)(item.e - lo);
            r.rev = true;
            r.layers = 1;
            r.bw = 2 * d + 1;
            r.klo0 = -d;
            r.vals = reinterpret_cast<int16_t *>(al_smem);
            r.rowm = reinterpret_cast<int16_t *>(al_smem + align_vals_bytes(1, r.bw));
            for (int k = lane; k < r.bw; k += 32) r.rowm[k] = kAlignInf;
            __syncwarp();
            align_sweep(r, lane);
            int best = -1;  // the largest column j of row m at d
            for (int k = lane; k < r.bw; k += 32) {
                const int j = m + r.klo0 + k;
                if (j >= 0 && j <= r.w && r.rowm[k] == d) best = max(best, j);
            }
            for (int o = 16; o; o >>= 1) best = max(best, __shfl_xor_sync(0xFFFFFFFFu, best, o));
            __syncwarp();
            if (best < 0) {
                if (lane == 0) align_put(out, item.idx, -1, -1, -1, -1, -1);
                continue;
            }
            s = item.e - best;
        }
        AlignSweep g{};
        g.P = P;
        g.T = H + s;
        g.m = m;
        g.w = (int)(item.e - s);
        g.generic = generic;
        if (generic) {
            g.layers = item.ins + 1;
            g.bw = item.dels + 1;
            g.klo0 = -(int)item.dels;
            g.S = item.subs;
            g.L = item.lim;
        } else {
            g.layers = 1;
            g.bw = align_lev_band(m, g.w, d, &g.klo0);
            if (g.bw == 0) {
                if (lane == 0) align_put(out, item.idx, -1, -1, -1, -1, -1);
                continue;
            }
        }
        g.vals = reinterpret_cast<int16_t *>(al_smem);
        g.table = reinterpret_cast<uint32_t *>(al_smem + align_vals_bytes(g.layers, g.bw));
        const uint32_t words = (uint32_t)(align_table_bytes(g.layers, m, g.bw) / 4);
        for (uint32_t q = lane; q < words; q += 32) g.table[q] = 0;
        __syncwarp();
        align_sweep(g, lane);
        if (lane == 0) {
            // the final cell: Levenshtein's one; generic: the smallest total over the layers, the fewest insertions
            const int R = (int)align_ring(g.bw), fin = (g.m + g.w) % 3;
            int lf = -1, c = kAlignInf;
            for (int l = 0; l < g.layers; l++) {
                const int klo = g.klo0 + (generic ? l : 0), k = g.w - m;
                if (k < klo || k > klo + g.bw - 1) continue;
                const int v = g.vals[(fin * g.layers + l) * R + m % R];
                if (v >= kAlignInf) continue;
                const int total = generic ? v + l + (l - k) : v;
                if (total < c) c = total, lf = l;
            }
            if (lf < 0 || c > d) {
                align_put(out, item.idx, -1, -1, -1, -1, -1);
            } else {
                // two walks back from (m, w): count, then write the ops in sequence order
                int x = 0, ni = 0, nd = 0;
                for (int pass = 0; pass < 2; pass++) {
                    int l = lf, i = m, j = g.w, pos = m + ni;
                    while (i > 0 || j > 0) {
                        const int klo = g.klo0 + (generic ? l : 0);
                        const uint64_t cell = ((uint64_t)l * (m + 1) + i) * g.bw + (j - i - klo);
                        const uint32_t code = (g.table[cell >> 4] >> (2 * (cell & 15))) & 3u;
                        uint8_t op;
                        if (code == 0) {
                            op = P[i - 1] != g.T[j - 1] ? 'X' : '=';
                            x += pass == 0 && op == 'X';
                            i--, j--;
                        } else if (code == 1) {
                            op = 'D';
                            nd += pass == 0;
                            i--;
                        } else {
                            op = 'I';
                            ni += pass == 0;
                            j--;
                            if (generic) l--;
                        }
                        if (pass == 1) out.ops[item.op_off + --pos] = op;
                    }
                }
                align_put(out, item.idx, s, x + ni + nd, x, ni, nd);
            }
        }
        __syncwarp();
    }
}

}  // namespace fzb
