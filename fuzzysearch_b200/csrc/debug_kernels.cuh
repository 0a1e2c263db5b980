// debug_kernels.cuh -- test-only entry into the expansion routines of the verify kernels
// (fzb_debug_expand): lets the reference's own _expand fixtures (tests/test_levenshtein.py:64-158
// TestExpandBase, and the recorded expand / expand_short / expand_long calls) run on the device directly
// instead of only through whole searches.
#pragma once
#include "kernels.cuh"

namespace fzb {

constexpr int kDbgMax = 256;

// One 32-thread block per case; thread 0 evaluates the case through the four device code paths:
//   out[0..1] bit-parallel, right-expansion form (sub = P[0:], seq walked forwards)
//   out[2..3] bit-parallel, left-expansion form  (sub = reversed P[:s], seq walked backwards)
//   out[4..5] cell-by-cell DP, forwards;  out[6..7] cell-by-cell DP, backwards
// (dist, len), (-1, -1) for (None, None), (-2, -2) where the path does not apply (bit-parallel: sub > 64).
__global__ void __launch_bounds__(32)
k_debug_expand(const uint8_t *subs, const uint32_t *sub_off, const uint8_t *seqs, const uint32_t *seq_off,
               const int32_t *max_l, const int32_t *variant, int32_t *out) {
    __shared__ uint8_t sSub[kDbgMax], sSubR[kDbgMax], sSeq[2 * kDbgMax], sSeqR[2 * kDbgMax];
    __shared__ unsigned long long sPM[256], sPMR[256];
    const uint32_t c = blockIdx.x;
    const int sublen = (int)(sub_off[c + 1] - sub_off[c]), seqlen = (int)(seq_off[c + 1] - seq_off[c]);
    for (int i = threadIdx.x; i < sublen; i += 32) {
        sSub[i] = subs[sub_off[c] + i];
        sSubR[sublen - 1 - i] = subs[sub_off[c] + i];
    }
    for (int i = threadIdx.x; i < seqlen; i += 32) {
        sSeq[i] = seqs[seq_off[c] + i];
        sSeqR[seqlen - 1 - i] = seqs[seq_off[c] + i];
    }
    __syncthreads();
    build_pm(sPM, sSub, sublen, threadIdx.x, 32);
    build_pm(sPMR, sSubR, sublen, threadIdx.x, 32);
    __syncthreads();
    if (threadIdx.x != 0) return;
    const int k = max_l[c], var = variant[c];
    int32_t *o = out + 8 * (size_t)c;
    int d = 0, l = 0;
    bool ok;
    if (sublen <= 64) {
        if (sublen <= 32)
            ok = expand_bp<uint32_t, 1>(EqPM<1>{sPM, 0}, sublen, sSeq, seqlen, k, d, l, var);
        else
            ok = expand_bp<unsigned long long, 1>(EqPM<1>{sPM, 0}, sublen, sSeq, seqlen, k, d, l, var);
        o[0] = ok ? d : -1;
        o[1] = ok ? l : -1;
        if (sublen <= 32)
            ok = expand_bp<uint32_t, -1>(EqPM<-1>{sPMR, sublen}, sublen, sSeqR + seqlen - 1, seqlen, k, d, l, var);
        else
            ok = expand_bp<unsigned long long, -1>(EqPM<-1>{sPMR, sublen}, sublen, sSeqR + seqlen - 1, seqlen, k, d,
                                                   l, var);
        o[2] = ok ? d : -1;
        o[3] = ok ? l : -1;
    } else {
        o[0] = o[1] = o[2] = o[3] = -2;
    }
    DpScratch S;
    const bool is_long = var == 2;  // (variant 0: expand_any picks it)
    if (var == 0)
        ok = expand_any<1>(sSub, sublen, sSeq, seqlen, k, S, d, l);
    else
        ok = expand_dp<1>(sSub, sublen, sSeq, seqlen, k, is_long, S, d, l);
    o[4] = ok ? d : -1;
    o[5] = ok ? l : -1;
    if (var == 0)
        ok = expand_any<-1>(sSubR + sublen - 1, sublen, sSeqR + seqlen - 1, seqlen, k, S, d, l);
    else
        ok = expand_dp<-1>(sSubR + sublen - 1, sublen, sSeqR + seqlen - 1, seqlen, k, is_long, S, d, l);
    o[6] = ok ? d : -1;
    o[7] = ok ? l : -1;
}

}  // namespace fzb
