"""The restatement the nearest-match tests compare with (test_gpu_nearest.nearest_E), checked without a device:
against a plain triple-loop table, against the per-segment scheme with its 2m warm-up, and against the oracle for the
premise find_nearest_matches rests on -- find_near_matches(P, S, max_l_dist=k) is non-empty iff k >= d* -- on all
three Levenshtein routes."""
import numpy as np

import oracle
from test_gpu_nearest import MIN_SEG, nearest, nearest_E, nearest_rows, seam_cases, segmented
from test_gpu_records import rand


def table_E(P, S):
    m, n = len(P), len(S)
    D = [[0] * (n + 1) for _ in range(m + 1)]
    for i in range(1, m + 1):
        D[i][0] = i
        for j in range(1, n + 1):
            D[i][j] = min(D[i - 1][j] + 1, D[i][j - 1] + 1, D[i - 1][j - 1] + (P[i - 1] != S[j - 1]))
    return D[m]


def test_restatement_equals_the_plain_table():
    rng = np.random.default_rng(1)
    for _ in range(300):
        alphabet = [b"ab", b"ACGT", b"abcdefgh"][int(rng.integers(0, 3))]
        P, S = rand(rng, alphabet, int(rng.integers(1, 12))), rand(rng, alphabet, int(rng.integers(0, 60)))
        assert nearest_E(P, S, block=int(rng.integers(1, 9))).tolist() == table_E(P, S), (P, S)
        E = nearest_E(P, S)
        assert E[0] == len(P) and E.max() <= len(P)
    rows = np.frombuffer(rand(rng, b"ab", 40 * 25), dtype=np.uint8).reshape(40, 25)
    d, e = nearest_rows(b"abbab", rows)
    assert [(int(a), int(b)) for a, b in zip(d, e)] == [nearest(b"abbab", bytes(r))[::2] for r in rows]


def test_a_warm_up_of_2m_is_exact_and_one_of_m_is_not():
    rng = np.random.default_rng(28)  # (as test_gpu_nearest: a seed whose cases hold a text the short warm-up fails on)
    wrong = 0
    for P, S in seam_cases(rng, 24, MIN_SEG, range(-4, 54)):
        assert segmented(P, S, MIN_SEG, 2 * len(P)) == nearest(P, S)
        wrong += segmented(P, S, MIN_SEG, len(P)) != nearest(P, S)
    assert wrong > 0
    for _ in range(60):
        P, S = rand(rng, b"ab", int(rng.integers(1, 9))), rand(rng, b"ab", int(rng.integers(0, 80)))
        assert segmented(P, S, int(rng.integers(1, 20)), 2 * len(P)) == nearest(P, S)


def test_a_match_exists_exactly_from_the_nearest_distance_on():
    """k == 0 (exact), len(P) // (k + 1) >= 3 (n-grams) and below (LP), small alphabets, k around d*."""
    rng = np.random.default_rng(2)
    routes = set()
    for _ in range(400):
        alphabet = [b"ab", b"abc", b"ACGT"][int(rng.integers(0, 3))]
        m = int(rng.integers(1, 16))
        P, S = rand(rng, alphabet, m), bytearray(rand(rng, alphabet, int(rng.integers(0, 120))))
        if rng.random() < 0.3 and len(S) >= m:
            S[5:5 + m] = P
        S = bytes(S)
        d = nearest(P, S)[0]
        routes.add("exact" if d == 0 else "ngrams" if m // (d + 1) >= 3 else "lp")
        assert oracle.find_near_matches(P, S, max_l_dist=d), (P, S, d)
        assert oracle.find_near_matches(P, S, max_l_dist=d + 1), (P, S, d)
        if d:
            assert not oracle.find_near_matches(P, S, max_l_dist=d - 1), (P, S, d)
            ms = oracle.find_near_matches(P, S, max_l_dist=d)
            assert min(x[2] for x in ms) == d
    assert routes == {"exact", "ngrams", "lp"}
