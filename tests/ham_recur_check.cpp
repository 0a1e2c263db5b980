// CPU check of the Hamming counting filter's recurrences (fuzzysearch_b200/csrc/ham_recur.h), exactly as
// k_hamming_count applies them: one "thread" per 128-byte row, 7 warm-up words from the previous row, candidates
// tracked over the row's own 32 words, flagged rows mark a range of start positions.  For random texts with
// planted near-matches, EVERY start p with Hamming(P, H[p:p+m]) <= k must fall inside a marked range -- with three
// slices, and with two slices where Wc - k <= 4.  Prints the number of flagged rows of each (selectivity).
// Build + run: tests/test_ham_recurrence.py (g++ -O2).
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>

#include "../fuzzysearch_b200/csrc/ham_recur.h"

using namespace fzb;

static uint64_t rng_state = 0x1234567ull;
static uint32_t rnd() {
    rng_state ^= rng_state << 13;
    rng_state ^= rng_state >> 7;
    rng_state ^= rng_state << 17;
    return (uint32_t)(rng_state >> 11);
}

struct Range {
    long lo, hi;
};

int main() {
    const char *alphabets[] = {"ACGT", "ab", "abcdefghijklmnopqrstuvwxyz"};
    long flagged_s = 0, checked = 0, rows_total = 0, flagged_2 = 0, flagged_s_two = 0, n_two = 0;
    for (int trial = 0; trial < 400; trial++) {
        const char *alpha = alphabets[trial % 3];
        const int alen = (int)strlen(alpha);
        const int k = (int)(rnd() % 8);
        const int m_min = 4 * k + 7;
        const int m = m_min + (int)(rnd() % (64 - m_min > 0 ? 64 - m_min : 1)) + (trial % 5 == 0 ? 60 : 0);
        const long n = 3000 + rnd() % 40000;
        std::vector<uint8_t> P(m), H(n);
        for (auto &c : P) c = (uint8_t)alpha[rnd() % alen];
        for (auto &c : H) c = (uint8_t)alpha[rnd() % alen];
        for (int t = 0; t < 40; t++) {  // plants with 0..k+1 substitutions, at every alignment, incl. both ends
            long pos = t == 0 ? 0 : (t == 1 ? n - m : (long)(rnd() % (n - m + 1)));
            std::vector<uint8_t> v(P);
            const int subs = (int)(rnd() % (k + 2));
            for (int s = 0; s < subs; s++) v[rnd() % m] = (uint8_t)alpha[rnd() % alen];
            memcpy(&H[pos], v.data(), m);
        }
        const int Wc = (m - 3) / 4 < 8 ? (m - 3) / 4 : 8;
        const int bias = 8 - (Wc - k);
        if (Wc - k < 1 || bias < 0 || bias > 7) {
            printf("bad parameters m=%d k=%d\n", m, k);
            return 1;
        }
        std::vector<uint32_t> Ts(kHcBuckets, 0u);  // the table
        for (int o0 = 0; o0 < 4; o0++)
            for (int i = 0; i < Wc; i++) Ts[hc_bucket(hc_gram(P.data(), o0 + 4 * i))] |= 1u << (8 * o0 + i);
        const long nrows = (n + 127) / 128;
        std::vector<uint8_t> buf((size_t)(nrows + 1) * 128 + 128, 0);  // row -1 (zeros) + rows + padding
        memcpy(&buf[128], H.data(), n);
        auto word = [&](long widx) -> uint32_t {  // widx relative to buffer start; row -1 = words -32..-1
            const uint8_t *q = &buf[128 + widx * 4];
            return (uint32_t)q[0] | ((uint32_t)q[1] << 8) | ((uint32_t)q[2] << 16) | ((uint32_t)q[3] << 24);
        };
        const uint32_t B0 = (bias & 1) ? 0x01010101u : 0u, B1 = (bias & 2) ? 0x01010101u : 0u,
                       B2 = (bias & 4) ? 0x01010101u : 0u;
        const bool two = Wc - k <= 4;  // the two-slice layout applies
        const int bias2 = 4 - (Wc - k);
        const uint32_t C0 = (two && (bias2 & 1)) ? 0x01010101u : 0u, C1 = (two && (bias2 & 2)) ? 0x01010101u : 0u;
        std::vector<Range> marks_s, marks_2;
        for (long r = 0; r < nrows; r++) {
            uint32_t acc_s = 0, acc_2 = 0;
            HamSliced cnt{0, 0, 0};
            HamSliced2 cnt2{0, 0};
            for (long t = r * 32 - 7; t < r * 32 + 32; t++) {
                const uint32_t w = word(t);
                const bool track = t >= r * 32;
                const uint32_t carry = ham_sliced_step(cnt, Ts[hc_bucket(w)], B0, B1, B2);
                if (track) acc_s |= carry;
                const uint32_t carry2 = two ? ham_sliced2_step(cnt2, Ts[hc_bucket(w)], C0, C1) : 0u;
                if (track) acc_2 |= carry2;
            }
            const long pr_lo = 4 * (r * 32 - Wc + 1) - 3;
            if (acc_s) marks_s.push_back({pr_lo < 0 ? 0 : pr_lo, 4 * (r * 32 + 31)});
            if (acc_2) marks_2.push_back({pr_lo < 0 ? 0 : pr_lo, 4 * (r * 32 + 31)});
        }
        if (two) {
            n_two++;
            flagged_2 += (long)marks_2.size();
            flagged_s_two += (long)marks_s.size();
        }
        flagged_s += (long)marks_s.size();
        rows_total += nrows;
        for (long p = 0; p + m <= n; p++) {
            int nd = 0;
            for (int i = 0; i < m && nd <= k; i++) nd += H[p + i] != P[i];
            if (nd > k) continue;
            checked++;
            bool in_s = false, in_2 = !two;
            for (auto &g : marks_s) in_s |= (p >= g.lo && p <= g.hi);
            for (auto &g : marks_2) in_2 |= (p >= g.lo && p <= g.hi);
            if (!in_s || !in_2) {
                printf("MISS trial=%d m=%d k=%d Wc=%d p=%ld three=%d two=%d\n", trial, m, k, Wc, p, in_s, in_2);
                return 1;
            }
        }
    }
    printf("ok: %ld true matches covered; flagged rows with three slices=%ld of %ld; two-slice layout in %ld trials: "
           "%ld flagged rows (three slices: %ld)\n", checked, flagged_s, rows_total, n_two, flagged_2, flagged_s_two);
    return 0;
}
