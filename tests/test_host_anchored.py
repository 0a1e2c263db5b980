"""The restatement the anchored tests compare with (test_gpu_anchored.anchored), checked without a device: against a
plain triple-loop table, against the mirror identity ('end' on (P, R) is 'start' on the reversed pair), in its
substitutions-only form, in the symbols it says a scan reads, and in the many-pattern reduction with its tie rules."""
import numpy as np

from test_gpu_anchored import anchored, prefix_row, reduce_patterns, symbols_read
from test_gpu_nearest import nearest
from test_gpu_records import rand


def lev(P, R):
    """A plain Levenshtein table"""
    D = [[i + j if i * j == 0 else 0 for j in range(len(R) + 1)] for i in range(len(P) + 1)]
    for i in range(1, len(P) + 1):
        for j in range(1, len(R) + 1):
            D[i][j] = min(D[i - 1][j] + 1, D[i][j - 1] + 1, D[i - 1][j - 1] + (P[i - 1] != R[j - 1]))
    return D[len(P)][len(R)]


def test_restatement_equals_the_plain_table():
    rng = np.random.default_rng(1)
    for _ in range(250):
        alphabet = [b"ab", b"ACGT", b"abcdefgh"][int(rng.integers(0, 3))]
        P, R = rand(rng, alphabet, int(rng.integers(1, 10))), rand(rng, alphabet, int(rng.integers(0, 30)))
        n = len(R)
        A = [lev(P, R[:e]) for e in range(n + 1)]
        B = [lev(P, R[s:]) for s in range(n + 1)]
        assert prefix_row(P, R).tolist() == A, (P, R)
        assert A[0] == len(P) and all(a >= e - len(P) for e, a in enumerate(A))
        d = min(A)
        assert anchored(P, R, "start") == (d, 0, A.index(d))
        d = min(B)
        assert anchored(P, R, "end") == (d, max(s for s in range(n + 1) if B[s] == d), n)
        # the mirror identity, and no window longer than 2m matters
        ds, s0, _ = anchored(P, R, "end")
        dm, _, e = anchored(P[::-1], R[::-1], "start")
        assert (ds, s0) == (dm, n - e)
        assert anchored(P, R[:2 * len(P)], "start") == anchored(P, R, "start")
        # anchored is never nearer than the free start
        assert anchored(P, R, "start")[0] >= nearest(P, R)[0]


def test_empty_records_ties_and_extremes():
    assert anchored(b"ACG", b"", "start") == (3, 0, 0) and anchored(b"ACG", b"", "end") == (3, 0, 0)
    assert anchored(b"A", b"AAA", "start") == (0, 0, 1)  # ties on e: the smallest
    assert anchored(b"A", b"AAA", "end") == (0, 2, 3)  # ties on s: the largest
    assert anchored(b"AA", b"XXXXXXX", "start") == (2, 0, 0)  # dist = m at e = 0
    assert anchored(b"AA", b"XXXXXXX", "end") == (2, 7, 7)
    assert symbols_read(b"ACGT", b"ACGTTTTTTTTT", "start") == 4  # dist 0 at e = 4: e = 5 cannot win
    assert symbols_read(b"AC", b"XXXXXXX", "start") == 3  # best 2 from e = 1 on: e = 4 cannot beat it
    assert symbols_read(b"AC", b"X", "end") == 1


def test_substitutions_only():
    rng = np.random.default_rng(2)
    for _ in range(200):
        P, R = rand(rng, b"ACGT", int(rng.integers(1, 12))), rand(rng, b"ACGT", int(rng.integers(0, 20)))
        m, n = len(P), len(R)
        for anchor in ("start", "end"):
            got = anchored(P, R, anchor, True)
            if n < m:
                assert got is None and symbols_read(P, R, anchor, True) == 0
                continue
            w = R[:m] if anchor == "start" else R[n - m:]
            assert got == (sum(a != b for a, b in zip(P, w)), 0 if anchor == "start" else n - m,
                           m if anchor == "start" else n)
            assert got[0] >= anchored(P, R, anchor)[0]  # (Levenshtein never costs more)


def test_many_pattern_reduction_and_ties():
    recs = [b"", b"AC", b"ACGT", b"GTAC", b"A"]
    pats = [b"ACG", b"AC", b"AC", b"TTTT"]
    for subs in (False, True):
        cols = reduce_patterns(pats, recs, "start", subs)
        for r, R in enumerate(recs):
            got = [(g[0], i) for i, P in enumerate(pats) for g in [anchored(P, R, "start", subs)] if g is not None]
            if not got:
                assert [c[r] for c in cols] == [-1] * 5
                continue
            d, i = min(got)
            assert (cols[0][r], cols[1][r]) == (i, d)
            rest = [x for x in got if x[1] != i]
            assert (cols[4][r], cols[3][r]) == (min(rest) if rest else (-1, -1))
    # pattern 1 and 2 are equal: the smaller index wins, the other is the runner-up
    cols = reduce_patterns(pats, [b"ACXX"], "start")
    assert (cols[0][0], cols[1][0], cols[2][0], cols[3][0], cols[4][0]) == (1, 0, 2, 2, 0)
    # under substitutions only a pattern longer than the record takes no part
    cols = reduce_patterns([b"ACGTA", b"GG"], [b"ACGT"], "end", True)
    assert [c[0] for c in cols] == [1, 1, 2, -1, -1]  # GG against GT
