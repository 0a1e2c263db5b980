// ham_recur.h -- the per-word recurrences of the Hamming counting filter (k_hamming_count), as plain
// functions usable from host code too (tests/ham_recur_check.cpp runs them on the CPU against brute force).
//
// For every 4-byte-aligned text word w and every alignment class o0 in {0,1,2,3} the filter keeps Wc <= 8
// counters: counter i (a "field") belongs to the occurrence whose FIRST counted word was seen i words ago and
// counts how many of its counted words so far equalled the pattern 4-gram at their own offset,
// P[o0+4j : o0+4j+4) for word j of the occurrence.  Per word: every field moves up by one, field 0 restarts
// at `bias`, and field i gets +1 iff w == gram(o0, i).
//
// The counters are bit-sliced: ONE 32-bit register per bit of the counters -- bit (8*o0 + i) of slice j is bit j
// of field i of class o0 -- so the table entry of a hash bucket is just the 32 match bits M (4 bytes: one LDS.32 =
// ONE shared-memory wavefront per warp and word when replicated per lane) and the increment is a ripple carry
// through the slices.  With three slices the fields count to 8 and bias = 8 - (Wc - k); the carry out of the top
// slice means ">= Wc - k of the occurrence's counted words match" -- a candidate, signalled at the word of the
// (Wc-k)-th match.  Thresholds Wc - k <= 4 need only two slices (fields count to 4, bias = 4 - (Wc - k)).
#pragma once
#include <stdint.h>

#if defined(__CUDACC__)
#define FZB_HD __host__ __device__ __forceinline__
#else
#define FZB_HD inline
#endif

namespace fzb {

constexpr uint32_t kHcHashMul = 0x9E3779B1u;
constexpr int kHcBuckets = 256;

FZB_HD uint32_t hc_bucket(uint32_t w) { return (w * kHcHashMul) >> 24; }

FZB_HD uint32_t hc_gram(const uint8_t *P, int o) {
    return (uint32_t)P[o] | ((uint32_t)P[o + 1] << 8) | ((uint32_t)P[o + 2] << 16) | ((uint32_t)P[o + 3] << 24);
}

struct HamSliced {
    uint32_t b0, b1, b2;
};

// B0..B2: bit j of `bias` replicated into field 0 of every class (0x01010101 or 0).  Returns the carry out
// of the counters: bit (8*o0 + i) set iff field i of class o0 just reached 8.
FZB_HD uint32_t ham_sliced_step(HamSliced &s, uint32_t M, uint32_t B0, uint32_t B1, uint32_t B2) {
    const uint32_t x0 = ((s.b0 + s.b0) & 0xFEFEFEFEu) | B0;  // fields move up, field 0 restarts at the bias
    const uint32_t x1 = ((s.b1 + s.b1) & 0xFEFEFEFEu) | B1;
    const uint32_t x2 = ((s.b2 + s.b2) & 0xFEFEFEFEu) | B2;
    const uint32_t c0 = x0 & M;                               // + M, rippling through the three slices
    s.b0 = x0 ^ M;
    const uint32_t c1 = x1 & c0;
    s.b1 = x1 ^ c0;
    s.b2 = x2 ^ c1;
    return x2 & c1;
}

// The same with TWO slices, for thresholds Wc - k <= 4: counters count to 4, bias = 4 - (Wc - k), and the
// carry out of slice 1 is the candidate signal -- four fewer ALU operations per word.
struct HamSliced2 {
    uint32_t b0, b1;
};

FZB_HD uint32_t ham_sliced2_step(HamSliced2 &s, uint32_t M, uint32_t B0, uint32_t B1) {
    const uint32_t x0 = ((s.b0 + s.b0) & 0xFEFEFEFEu) | B0;
    const uint32_t x1 = ((s.b1 + s.b1) & 0xFEFEFEFEu) | B1;
    const uint32_t c0 = x0 & M;
    s.b0 = x0 ^ M;
    s.b1 = x1 ^ c0;
    return x1 & c0;
}

}  // namespace fzb
