// generic_batch_kernels.cuh -- the verification kernels of batches of generic-limit patterns (DESIGN.md section 5.9).
//
// A generic pattern has per-operation limits tighter than its total (max_substitutions, max_insertions,
// max_deletions, max_l_dist).  Its candidates are found by the same shared scans as the Levenshtein batch's
// (batch_kernels.cuh): both routes of the single generic search use those filters with k = max_l_dist, so they are
// admissible for generic limits too.  Only the verification differs -- the generic NFA sim_generic
// (generic_search.py:57-177) with each pattern's own limits, read from a per-pattern table
// (subs | ins << 8 | dels << 16) next to the BatchPat array:
//   k_verify_multi_generic     the (pattern, granule) work items of k_filter_multi, one warp per item: the same
//                              verify_granule_generic as the single n-gram route (k_verify_generic).
//   k_verify_mhits_generic     the (pattern, n-gram j, idx) hits of k_filter_mdense, one warp per hit: the search
//                              window test (generic_search.py:223-227), the window [p0-k, p0+m+k) staged in shared
//                              memory, its starts split across the lanes -- what verify_granule_generic does for
//                              one hit.
//   k_lp_verify_multi_generic  the survivors of k_lp_scan_multi -> k_lm_refine -> k_lm_scatter (LP route), one per
//                              lane: sim_generic straight away (the bit-parallel automaton of k_lp_verify_multi
//                              models no per-operation limits).
// Each lane's two candidate lists come from the scratch slab, `cap` entries each; a start with more live candidates
// raises CNT_OVERFLOW and the host searches the pass's patterns one by one.  Records carry pattern << 8 | n-gram
// (n-gram routes) or pattern << 8 | 1 (LP route), as in the other batches.  All three declare one CTA per SM as
// their minimum: with the default bound ptxas holds them at 40-48 registers and spills the NFA's state.
#pragma once
#include "batch_kernels.cuh"

namespace fzb {

struct GenericCtx {  // what sim_generic and verify_granule_generic need, per pattern
    const uint8_t *H;
    int64_t buf_lo, buf_len, N, own_lo, own_hi;
    int32_t m, k, L, n_ngrams;
    int32_t max_subs, max_ins, max_dels;
};

__device__ __forceinline__ void generic_ctx_geometry(GenericCtx &c, const uint8_t *H, int64_t buf_lo, int64_t buf_len,
                                                     int64_t N, int64_t own_lo, int64_t own_hi) {
    c.H = H;
    c.buf_lo = buf_lo;
    c.buf_len = buf_len;
    c.N = N;
    c.own_lo = own_lo;
    c.own_hi = own_hi;
    c.m = 1;
    c.k = c.L = c.n_ngrams = 0;
    c.max_subs = c.max_ins = c.max_dels = 0;
}

// the pattern's lengths from its BatchPat, its limits from the table
__device__ __forceinline__ void generic_ctx_pattern(GenericCtx &c, const BatchPat *bp, const uint32_t *glim, uint32_t pid) {
    c.m = bp->m;
    c.k = bp->k;
    c.L = bp->L;
    c.n_ngrams = bp->n_ngrams;
    const uint32_t g = __ldg(glim + pid);
    c.max_subs = (int)(g & 0xFFu);
    c.max_ins = (int)((g >> 8) & 0xFFu);
    c.max_dels = (int)((g >> 16) & 0xFFu);
}

// REC (all three kernels): the handle holds a record set `rs`; every window and NFA run stays inside the record of
// its anchor or start, as in the single generic search (k_verify_generic, k_generic_lp).  REC == false never reads rs.
template <bool REC>
__global__ void __launch_bounds__(kLpThreads, 1)
k_verify_multi_generic(const __grid_constant__ MultiParams p, const BatchPat *pats, const uint32_t *glim,
                       uint32_t *scratch, int cap, RawRec *out, uint32_t ocap, uint32_t *counters, const RecSet rs) {
    __shared__ __align__(8) uint8_t sPall[kLpThreads / 32][kBatchMaxM];
    __shared__ uint32_t sWinAll[kLpThreads / 32][kWinWords];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    uint8_t *sP = sPall[warp];
    uint32_t *sWin = sWinAll[warp];
    const int64_t tid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    uint32_t *A = scratch + tid * 2 * (int64_t)cap, *B = A + cap;
    const uint32_t nitems = min(counters[CNT_GRAN], p.work_cap);
    uint32_t cur_pid = 0xFFFFFFFFu;
    GenericCtx c;
    generic_ctx_geometry(c, p.H, p.buf_lo, p.buf_len, p.N, p.own_lo, p.own_hi);
    for (;;) {
        uint32_t item = 0;
        if (lane == 0) item = atomicAdd(&counters[CNT_WORK], 1u);
        item = __shfl_sync(0xFFFFFFFFu, item, 0);
        if (item >= nitems) break;
        const WorkItem it = p.work[item];
        if (it.pid != cur_pid) {  // load the pattern and its limits
            const BatchPat *bp = pats + it.pid;
            __syncwarp();
            if (lane < kBatchMaxM / 4) reinterpret_cast<uint32_t *>(sP)[lane] = reinterpret_cast<const uint32_t *>(bp->P)[lane];
            generic_ctx_pattern(c, bp, glim, it.pid);
            __syncwarp();
            cur_pid = it.pid;
        }
        if constexpr (REC)
            verify_granule_generic_rec(c, sP, sWin, (int64_t)it.granule, lane, A, B, cap, out, ocap, counters, rs,
                                       (int)(it.pid << 8));
        else
            verify_granule_generic(c, sP, sWin, (int64_t)it.granule, lane, A, B, cap, out, ocap, counters, (int)(it.pid << 8));
        if (lane == 0) p.set[it.slot] = 0ull;  // the set is empty again when the kernel ends
    }
    if (blockIdx.x == 0 && threadIdx.x == 0) atomicAdd(&counters[CNT_CAND], nitems);
}

// A warp's window slot: [p0-k, p0+m+k) starts on a 4-byte boundary and is copied in whole words, so it needs
// m + 2k + 6 bytes; the host admits a pattern when m + 2k + 8 <= kMhgSlotBytes.
constexpr int kMhgSlotBytes = 128;

template <bool REC>
__global__ void __launch_bounds__(kLpThreads, 1)
k_verify_mhits_generic(const __grid_constant__ MdenseParams p, const uint32_t *glim, uint32_t *scratch, int cap,
                       RawRec *out, uint32_t ocap, uint32_t *counters, const RecSet rs) {
    __shared__ __align__(8) uint8_t sPall[kLpThreads / 32][kBatchMaxM];
    __shared__ uint32_t sWinAll[kLpThreads / 32][kMhgSlotBytes / 4];
    const uint32_t nhits = counters[CNT_MHITS];
    if (nhits > p.hits_cap) {  // list overflowed: the host searches these patterns one by one
        if (blockIdx.x == 0 && threadIdx.x == 0) counters[CNT_OVERFLOW] = 1;
        return;
    }
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    uint8_t *sP = sPall[warp];
    uint32_t *sWin = sWinAll[warp];
    const int64_t tid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    uint32_t *A = scratch + tid * 2 * (int64_t)cap, *B = A + cap;
    const MultiParams &mp = p.mp;
    GenericCtx c;
    generic_ctx_geometry(c, mp.H, mp.buf_lo, mp.buf_len, mp.N, mp.own_lo, mp.own_hi);
    const int64_t N = mp.N;
    for (;;) {
        uint32_t item = 0;
        if (lane == 0) item = atomicAdd(&counters[CNT_MHITWORK], 1u);
        item = __shfl_sync(0xFFFFFFFFu, item, 0);
        if (item >= nhits) break;
        const unsigned long long hv = p.hits[item];
        const int64_t idx = mp.buf_lo + (int64_t)(hv & ((1ull << 40) - 1));
        const int j = (int)((hv >> 40) & 0xFFu);
        const uint32_t pid = (uint32_t)(hv >> 48);
        const BatchPat *bp = p.pats + pid;
        generic_ctx_pattern(c, bp, glim, pid);
        const int m = c.m, k = c.k, L = c.L, s = j * L;
        int64_t wlo, whi;
        if constexpr (REC) {  // the same arithmetic with the hit's own record [lo, hi) for [0, N); a separator is dropped
            int64_t lo, hi;
            if (!rec_bounds(rs, idx, lo, hi)) continue;
            int64_t ws = lo + max((int64_t)0, (int64_t)(s - k));
            int64_t we = min(hi, hi - m + s + L + k);
            if (we <= ws) continue;
            ws = max(lo, min(ws, hi));
            we = max(ws, min(we, hi));
            if (idx < ws || idx + L > we) continue;
            wlo = max(lo, idx - s - k);
            whi = min(hi, idx - s + m + k);
        } else {
            // the search window of n-gram j (generic_search.py:223-227); the filter already checked the n-gram itself
            int64_t ws = max((int64_t)0, (int64_t)(s - k));
            int64_t we = min(N, N - m + s + L + k);
            if (we <= ws) continue;
            ws = max((int64_t)0, min(ws, N));
            we = max(ws, min(we, N));
            if (idx < ws || idx + L > we) continue;
            const int64_t p0 = idx - s;
            wlo = max((int64_t)0, p0 - k);  // :231
            whi = min(N, p0 + m + k);
        }
        const int64_t alo = max(wlo, mp.buf_lo) & ~(int64_t)3;  // buf_lo is a multiple of 16
        const int nwords = (int)((min(whi, mp.buf_lo + mp.buf_len) - alo + 3) >> 2);
        const uint32_t *src = reinterpret_cast<const uint32_t *>(mp.H + (alo - mp.buf_lo));
        __syncwarp();  // the previous hit's lanes are done with the slot and the pattern
        if (lane < kBatchMaxM / 4) reinterpret_cast<uint32_t *>(sP)[lane] = __ldg(reinterpret_cast<const uint32_t *>(bp->P) + lane);
        for (int w = lane; w < nwords; w += 32) sWin[w] = __ldg(src + w);  // padded buffer
        __syncwarp();
        const uint8_t *W = reinterpret_cast<const uint8_t *>(sWin) - alo;  // W[g]: byte at global g
        for (int64_t st = wlo + lane; st < whi; st += 32)
            if (!sim_generic(c, sP, W, st, whi, A, B, cap, idx, j | (int)(pid << 8), out, ocap, counters))
                atomicExch(&counters[CNT_OVERFLOW], 1u);
    }
    if (blockIdx.x == 0 && threadIdx.x == 0) atomicAdd(&counters[CNT_CAND], nhits);
}

// One survivor per lane; a lane that is done takes the next one (its own atomic on the work counter), so lanes whose
// NFA dies early do not wait for the rest of the warp before they refill.  The survivors are grouped by pattern
// (k_lm_scatter), so neighbouring lanes mostly run the same pattern.
template <bool REC>
__global__ void __launch_bounds__(kLpThreads, 1)
k_lp_verify_multi_generic(const __grid_constant__ LpMultiParams p, const uint32_t *glim, const unsigned long long *sorted,
                          const uint32_t *hist, uint32_t *scratch, int cap, RawRec *out, uint32_t ocap,
                          uint32_t *counters, const RecSet rs) {
    __shared__ __align__(4) uint8_t sPat[kLpThreads][kBatchMaxM / 2];  // LP patterns are at most 31 bytes
    if (counters[CNT_LMLIST] > p.list_cap) {  // the scan's list overflowed: the host searches these patterns one by one
        if (blockIdx.x == 0 && threadIdx.x == 0) counters[CNT_LMWORK] = 1;
        return;
    }
    const uint32_t n = hist[64];  // exact survivors, grouped by pattern
    const int64_t tid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    uint32_t *A = scratch + tid * 2 * (int64_t)cap, *B = A + cap;
    const uint8_t *W = p.H - p.buf_lo;  // W[g]: byte at global position g
    uint8_t *myP = sPat[threadIdx.x];
    GenericCtx c;
    generic_ctx_geometry(c, p.H, p.buf_lo, p.buf_len, p.N, p.own_lo, p.own_hi);
    uint32_t cur_pid = 0xFFFFFFFFu;
    for (;;) {
        const uint32_t idx = atomicAdd(&counters[CNT_LMNEXT], 1u);
        if (idx >= n) break;
        const unsigned long long ent = sorted[idx];
        const int64_t st = p.buf_lo + (int64_t)(ent & ((1ull << 40) - 1));
        const uint32_t pid = (uint32_t)(ent >> 40);
        if (pid != cur_pid) {
            const BatchPat *bp = p.pats + pid;
            for (int w = 0; w < kBatchMaxM / 8; w++)
                reinterpret_cast<uint32_t *>(myP)[w] = __ldg(reinterpret_cast<const uint32_t *>(bp->P) + w);
            generic_ctx_pattern(c, bp, glim, pid);
            cur_pid = pid;
        }
        int64_t lo = 0, seq_end = p.N;
        if (REC && !rec_bounds(rs, st, lo, seq_end)) continue;  // a separator is no start
        if (!sim_generic(c, myP, W, st, seq_end, A, B, cap, st, 1 | (int)(pid << 8), out, ocap, counters))
            atomicExch(&counters[CNT_OVERFLOW], 1u);
    }
    if (blockIdx.x == 0 && threadIdx.x == 0) atomicAdd(&counters[CNT_CAND], counters[CNT_LMLIST]);
}

}  // namespace fzb
