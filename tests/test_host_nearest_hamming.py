"""The restatement the substitutions-only nearest tests compare with (test_gpu_nearest_hamming.hamming_H), checked
without a device: against a plain double loop, against the per-segment scheme with its m - 1 warm-up and end gating,
and against the oracle for the premise find_nearest_matches(..., substitutions_only=True) rests on --
find_near_matches(P, S, max_substitutions=k, max_insertions=0, max_deletions=0) lists exactly the windows with at most
k mismatches -- on the exact, n-gram and LP substitution routes."""
import numpy as np

import oracle
from test_gpu_nearest_hamming import hamming, hamming_H, hamming_rows
from test_gpu_records import rand


def plain_H(P, S):
    m, n = len(P), len(S)
    return [sum(P[j] != S[e - m + j] for j in range(m)) for e in range(m, n + 1)]


def segmented(P, S, seg, warm, base=0):
    """The per-segment scheme of k_nearest_hamming_scan transcribed on the host: every segment of `seg` bytes is
    scanned by a fresh column started `warm` bytes before it (never before the record start `base`), a column tracks
    an end only once it has read m bytes since its reset, and only the ends inside the segment count."""
    m, n = len(P), len(S)
    best = None
    for a in range(base, n, seg):
        w = max(a - warm, base)
        fill = m - 1  # bytes the column still needs after its reset
        for x in range(w, min(a + seg, n)):
            if fill:
                fill -= 1
                continue
            if x < a:
                continue
            e = x + 1
            h = sum(P[j] != S[e - m + j] for j in range(m))
            if best is None or h < best[0]:
                best = [h, 1, e]
            elif h == best[0]:
                best[1] += 1
    return None if best is None else tuple(best)


def test_restatement_equals_the_plain_loop():
    rng = np.random.default_rng(81)
    for _ in range(300):
        alphabet = [b"ab", b"ACGT", b"abcdefgh"][int(rng.integers(0, 3))]
        P, S = rand(rng, alphabet, int(rng.integers(1, 12))), rand(rng, alphabet, int(rng.integers(0, 60)))
        assert hamming_H(P, S).tolist() == plain_H(P, S), (P, S)
        H = plain_H(P, S)
        assert hamming(P, S) == (None if not H else (min(H), H.count(min(H)), H.index(min(H)) + len(P)))
    rows = np.frombuffer(rand(rng, b"ab", 40 * 25), dtype=np.uint8).reshape(40, 25)
    d, e = hamming_rows(b"abbab", rows)
    assert [(int(a), int(b)) for a, b in zip(d, e)] == [hamming(b"abbab", bytes(r))[::2] for r in rows]
    d, e = hamming_rows(b"a" * 30, rows)
    assert d.tolist() == [-1] * 40 and e.tolist() == [-1] * 40


def test_a_warm_up_of_m_minus_1_with_gating_is_exact_and_one_of_m_minus_2_is_not():
    """Seam cases: the best window ends at every offset around a segment seam, up to m - 1 bytes behind it."""
    rng = np.random.default_rng(82)
    wrong = 0
    seg = 64
    for m in (1, 2, 5, 13):
        for o in range(-2, m + 3):
            P = rand(rng, b"ab", m)
            S = bytearray(b"c" * (3 * seg))
            S[seg + o - m:seg + o] = P
            S = bytes(S)
            assert segmented(P, S, seg, m - 1) == hamming(P, S), (m, o)
            if m >= 2:
                wrong += segmented(P, S, seg, m - 2) != hamming(P, S)
    assert wrong > 0
    for _ in range(80):
        P, S = rand(rng, b"ab", int(rng.integers(1, 9))), rand(rng, b"ab", int(rng.integers(0, 80)))
        assert segmented(P, S, int(rng.integers(1, 20)), len(P) - 1) == hamming(P, S), (P, S)
    # a record that starts inside the text: no window reaches behind its start
    S = b"GATTACA" + b"xGATTAC"
    assert segmented(b"GATTACA", S, 3, 6, base=8) == hamming(b"GATTACA", S[8:]) is None


def test_the_list_at_the_nearest_distance_is_exactly_its_windows():
    """k == 0 (exact), len(P) // (k + 1) >= 3 (n-grams) and below (LP), small alphabets: the list at d* has n_ends
    entries, the first ending at first_end; the list at d* - 1 is empty; n < m gives no list at any k."""
    rng = np.random.default_rng(83)
    routes = set()
    for _ in range(400):
        alphabet = [b"ab", b"abc", b"ACGT"][int(rng.integers(0, 3))]
        m = int(rng.integers(1, 16))
        P, S = rand(rng, alphabet, m), bytearray(rand(rng, alphabet, int(rng.integers(0, 120))))
        if rng.random() < 0.3 and len(S) >= m + 5:
            S[5:5 + m] = P
            S[5 + int(rng.integers(0, m))] = ord("x") if rng.random() < 0.5 else S[5]
        S = bytes(S)
        got = hamming(P, S)
        if got is None:
            for k in (0, 1, m):
                assert oracle.find_near_matches(P, S, max_substitutions=k, max_insertions=0, max_deletions=0) == []
            continue
        d, n_ends, first = got
        routes.add("exact" if d == 0 else "ngrams" if m // (d + 1) >= 3 else "lp")
        ms = oracle.find_near_matches(P, S, max_substitutions=d, max_insertions=0, max_deletions=0)
        assert len(ms) == n_ends and ms[0][1] == first and ms[0][0] == first - m, (P, S, d)
        assert all(x[2] == d for x in ms), (P, S, d)
        if d:
            assert oracle.find_near_matches(P, S, max_substitutions=d - 1, max_insertions=0, max_deletions=0) == []
    assert routes == {"exact", "ngrams", "lp"}
