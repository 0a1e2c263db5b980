"""The tile, buffer and chunk geometry of the five shared batch scans replayed on the emulated build: the bodies of the
-m gpu tests of test_gpu_batch_scans.py with the emulated grid (2 SMs) in place of the H100's.

Before that, the restatements those tests compare with are checked on their own, without a device: every true match
of every pattern lies behind a restated candidate (a marked granule, an n-gram hit, a key hit, an LP survivor), and
the numpy LP restatement equals a line-by-line transcription of k_lp_scan_multi's six-slice ripple counter.  A
mismatch on the device then points at the device."""
import numpy as np

import oracle
import test_gpu_batch_scans as G
from corpus import ASCII, DNA
from test_emu_kernels import emu_device, emu_lib  # noqa: F401  (fixtures)

M64 = (1 << 64) - 1


def planted(rng, alphabet, n, pats, ks, subs_only=False):
    hay = G.rand(rng, alphabet, n)
    G.plant_copies(rng, hay, pats, ks, alphabet, max(40, n // 30), subs_only)
    G.put(hay, 0, pats[0])
    G.put(hay, n - len(pats[-1]), pats[-1])
    return hay


def covered(count, pat, k, hay, lo, hi):
    """the restatement `count` has a candidate of the pattern alone with own range [lo, hi)"""
    return count([pat], [k], hay, 0, len(hay), lo, hi) > 0


def test_restatements_cover_every_match():
    """Every oracle match (s, e, d): the q-sample pass marks the granule of s (an aligned word inside the match equals
    a 4-gram P[o:o+4] with |g - o - s| <= k); an n-gram of P occurs intact in H[s:e] (k + 1 disjoint n-grams, k
    edits); a piece of P has a key hit at s + jL (pigeonhole over substitutions); s is an LP survivor."""
    rng = np.random.default_rng(701)
    checked = 0
    for trial in range(24):
        alphabet = (ASCII, DNA, b"abcdef")[trial % 3]
        n = int(rng.integers(300, 3000))
        # q-sample and prefix / 2-bit (Levenshtein, n-gram route)
        pats, ks = (G.qsample_mix if trial % 2 else G.prefix_mix)(rng)
        pats = [bytes(G.rand(rng, alphabet, len(p))) for p in pats]
        hay = planted(rng, alphabet, n, pats, ks)
        for p, k in zip(pats, ks):
            L = len(p) // (k + 1)
            sampled = (len(p) - k - 3) // 4 >= k + 1
            marked = G.qsample_granules([p], [k], hay, 0, 0, n)[0] if sampled else None
            for s, e, _ in oracle.levenshtein_raw(p, bytes(hay), k):
                assert covered(G.ngram_hits, p, k, hay, s, e - L + 1), (trial, p, k, s, e)
                if sampled:
                    assert (s >> 6) in marked, (trial, p, k, s)
                checked += 1
        # Hamming, text and 2-bit keys
        pats, ks = G.ham_text_mix(rng) if alphabet != DNA else G.ham_2bit_mix(rng)
        pats = [bytes(G.rand(rng, alphabet, len(p))) for p in pats]
        hay = planted(rng, alphabet, n, pats, ks, subs_only=True)
        for p, k in zip(pats, ks):
            for s, _, _ in oracle.substitutions(p, bytes(hay), k):
                assert G.ham_key_hits([p], [k], hay, 0, n, s, s + 1) > 0, (trial, p, k, s)
                assert G.ham_key_hits([p], [k], hay, 0, n, s, s + 1, two_bit=True) > 0, (trial, p, k, s)
                checked += 1
        # LP, Levenshtein and generic
        pats, ks = G.lp_mix(rng)
        pats = [bytes(G.rand(rng, alphabet, len(p))) for p in pats]
        hay = planted(rng, alphabet, n, pats, ks)
        for p, k in zip(pats, ks):
            for s, _, _ in oracle.levenshtein_raw(p, bytes(hay), k):
                assert G.lp_survivors(pats, ks, hay, 0, n, s, s + 1) > 0, (trial, p, k, s)
                checked += 1
            for s, _, _ in oracle.generic_raw(p, bytes(hay), k, k, k, k):
                assert G.lp_survivors(pats, ks, hay, 0, n, s, s + 1, generic=True) > 0, (trial, p, k, s)
    assert checked > 1000


def kernel_lp(pats, ks, buf, buf_lo, N, own_lo, own_hi, generic=False):
    """k_lp_scan_multi's survivors, one run of 128 starts at a time as its threads walk them: the lookup vectors A
    (byte in P) and F (byte may open P), six bit slices C[i] of bias + count per pattern, the first window counted
    byte by byte, then the slide (the byte at s leaves, the byte at s + wmax enters) as a ripple of up / down carries."""
    A, Fv = [0] * 256, [0] * 256
    bias = [0] * 6
    wmax = 0
    for i, (P, k) in enumerate(zip(pats, ks)):
        m = len(P)
        for c in P:
            A[c] |= 1 << i
        for c in (range(256) if generic else P[:min(k, m - 1) + 1]):
            Fv[c] |= 1 << i
        for b in range(6):
            if ((32 - (m - k)) >> b) & 1:
                bias[b] |= 1 << i
        wmax = max(wmax, m + k)
    H = bytes(buf)
    hi = min(own_hi, N)
    lim = min(N, buf_lo + len(H))
    byte = lambda g: H[g - buf_lo] if buf_lo <= g < buf_lo + len(H) else 0
    base = own_lo & ~127
    n = 0
    for s0 in range(base, hi, 128):
        C = list(bias)
        for j in range(wmax):
            carry = A[byte(s0 + j)] if s0 + j < lim else 0
            for i in range(6):
                c = C[i]
                C[i] = c ^ carry
                carry &= c
        for r in range(128):
            s = s0 + r
            la, lf = (A[byte(s)], Fv[byte(s)]) if s < lim else (0, 0)
            surv = C[5] & lf
            if surv and own_lo <= s < hi:
                n += bin(surv).count("1")
            ae = A[byte(s + wmax)] if s + wmax < lim else 0
            up, dn = ae & ~la & M64, la & ~ae & M64
            for i in range(6):
                c = C[i]
                C[i] = c ^ up ^ dn
                up &= c
                dn &= ~c & M64
    return n


def test_lp_restatement_equals_the_ripple_counter():
    """Random small inputs and LP mixes (need 1 to 15, wmax up to 31), own ranges off the 128-byte runs, buffers that
    start at buf_lo != 0 and end before N, Levenshtein and generic first bytes."""
    rng = np.random.default_rng(702)
    for trial in range(40):
        alphabet = (ASCII, DNA, b"abc", b"ab\0")[trial % 4]
        npat = int(rng.integers(2, 7))
        pats, ks = [], []
        for _ in range(npat):
            k = int(rng.integers(1, 9))
            m = int(rng.integers(k + 1, min(3 * k + 3, 31 - k) + 1))
            pats.append(bytes(G.rand(rng, alphabet, m)))
            ks.append(k)
        n = int(rng.integers(50, 700))
        buf_lo = 16 * int(rng.integers(0, 40))
        hay = planted(rng, alphabet, n, pats, ks)
        N = buf_lo + n + int(rng.integers(0, 2)) * int(rng.integers(1, 50))
        own_lo = buf_lo + int(rng.integers(0, n // 2))
        own_hi = own_lo + int(rng.integers(1, n))
        for generic in (False, True):
            want = kernel_lp(pats, ks, hay, buf_lo, N, own_lo, own_hi, generic)
            assert G.lp_survivors(pats, ks, hay, buf_lo, N, own_lo, own_hi, generic) == want, (trial, generic)
    # need = 1 in a pass of wmax = 31, a run of a pattern's bytes across a 128-byte run seam and to the buffer's end
    pats, ks = [b"ab", b"cdefghijklmnopqrstuvw"[:23 - 2] + b"xy", b"qz"], [1, 8, 1]
    hay = G.rand(np.random.default_rng(703), b"ABCDEFGH", 600)
    G.put(hay, 120, pats[1])
    G.put(hay, 600 - 15, pats[1])
    for own in ((0, 600), (100, 300), (127, 129), (500, 600)):
        assert G.lp_survivors(pats, ks, hay, 0, 600, *own) == kernel_lp(pats, ks, hay, 0, 600, *own), own


def test_emu_batch_scans_lengths(emu_device):
    G.test_qsample_lengths(emu_device, small=True)
    G.test_prefix_lengths(emu_device, small=True)
    G.test_two_bit_lengths(emu_device, small=True)


def test_emu_batch_scans_ham_lp(emu_device):
    G.test_ham_lengths(emu_device, small=True)
    G.test_lp_lengths(emu_device, small=True)
    G.test_generic_passes(emu_device, small=True)


def test_emu_batch_scans_edges(emu_device):
    G.test_nul_grams_and_reupload(emu_device, small=True)
    G.test_packed_tiles(emu_device, small=True)
    G.test_hash_collisions(emu_device, small=True)


def test_emu_batch_scans_geometry(emu_device):
    G.test_shards(emu_device, small=True)
    G.test_record_sets(emu_device, small=True)
    G.test_tiny_chunks(emu_device, small=True)
