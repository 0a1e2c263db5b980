"""The alignment rules of fzb_align / align_matches / align_in_each (DESIGN.md section 5.17) restated as plain Python
over the full table, and the restatement checked against brute force that enumerates every alignment of patterns and
windows of up to 6 symbols.  tests/test_gpu_align.py compares the device with `align_anchored` and `free_start`."""
import itertools
import random

import numpy as np
import pytest

from fuzzysearch_b200.search import _cigars

BIG = 1 << 29
INF = float("inf")
SMEM_MAX = 64 * 1024  # align_kernels.cuh: kAlignSmemMax


def classify(subs, ins, dels, l):
    """choose_search_class's rule on normalised limits (None already replaced by BIG)"""
    if l == 0:
        return "exact"
    if ins == 0 and dels == 0:
        return "hamming"
    if l <= min(subs, ins, dels):
        return "levenshtein"
    return "generic"


def cigar(ops):
    return "".join("%d%s" % (len(list(g)), c) for c, g in itertools.groupby(ops))


def align_anchored(P, T, limits, d):
    """The canonical alignment of P against the window T under the class of `limits` = (S, I, D, L) at a cost of at
    most d -> (cost, ops) or None.  Ops in sequence order: '=', 'X', 'I' (a symbol of T with no counterpart in P),
    'D' (a symbol of P missing from T)."""
    S, I, D, L = limits
    cls = classify(*limits)
    m, w = len(P), len(T)
    if cls in ("exact", "hamming"):
        assert w == m
        x = sum(a != b for a, b in zip(P, T))
        bound = 0 if cls == "exact" else min(d, S, L, m)
        return (x, "".join("=" if a == b else "X" for a, b in zip(P, T))) if x <= bound else None
    bound = min(d, L, max(m, w))
    if cls == "levenshtein":
        # full Levenshtein table, then the walk back from (m, w): diagonal, else D, else I
        V = [[INF] * (w + 1) for _ in range(m + 1)]
        for i in range(m + 1):
            for j in range(w + 1):
                if i == 0 and j == 0:
                    V[i][j] = 0
                    continue
                V[i][j] = min(V[i - 1][j - 1] + (P[i - 1] != T[j - 1]) if i and j else INF,
                              V[i - 1][j] + 1 if i else INF, V[i][j - 1] + 1 if j else INF)
        if V[m][w] > bound:
            return None
        ops, i, j = [], m, w
        while i or j:
            if i and j and V[i - 1][j - 1] + (P[i - 1] != T[j - 1]) == V[i][j]:
                ops.append("=" if P[i - 1] == T[j - 1] else "X")
                i, j = i - 1, j - 1
            elif i and V[i - 1][j] + 1 == V[i][j]:
                ops.append("D")
                i -= 1
            else:
                ops.append("I")
                j -= 1
        return V[m][w], "".join(reversed(ops))
    # generic: layer l = insertions used; a cell holds the fewest substitutions of a path reaching it with l
    # insertions and i - j + l deletions, within X <= S, D <= D_max and a total <= bound
    Ip, Dp, Sp = min(I, bound), min(D, bound), min(S, bound, m)
    X = [[[INF] * (w + 1) for _ in range(m + 1)] for _ in range(Ip + 1)]
    for l in range(Ip + 1):
        for i in range(m + 1):
            for j in range(w + 1):
                dl = i - j + l
                if dl < 0 or dl > Dp:
                    continue
                if i == 0 and j == 0:
                    X[l][i][j] = 0 if l == 0 else INF
                    continue
                v = min(X[l][i - 1][j - 1] + (P[i - 1] != T[j - 1]) if i and j else INF,
                        X[l][i - 1][j] if i else INF, X[l - 1][i][j - 1] if j and l else INF)
                X[l][i][j] = INF if v > Sp or v + l + dl > bound else v
    best = None
    for l in range(Ip + 1):
        dl = m - w + l
        if 0 <= dl <= Dp and X[l][m][w] < INF:
            total = X[l][m][w] + l + dl
            if best is None or total < best[0]:
                best = (total, l)
    if best is None:
        return None
    ops, l, i, j = [], best[1], m, w
    while i or j:
        if i and j and X[l][i - 1][j - 1] + (P[i - 1] != T[j - 1]) == X[l][i][j]:
            ops.append("=" if P[i - 1] == T[j - 1] else "X")
            i, j = i - 1, j - 1
        elif i and i - 1 - j + l >= 0 and X[l][i - 1][j] == X[l][i][j]:
            ops.append("D")
            i -= 1
        else:
            ops.append("I")
            j, l = j - 1, l - 1
    return best[0], "".join(reversed(ops))


def lev(P, T):
    return align_anchored(P, T, (BIG, BIG, BIG, BIG), BIG)[0]


def free_start(P, S, e, lo, limits, d):
    """The start of a free-start item ending at e in a record starting at lo -> s or None: substitutions only e - m;
    Levenshtein the smallest s in [max(lo, e - m - d), e] with lev(P, S[s:e]) == d."""
    m = len(P)
    if classify(*limits) == "hamming":
        return e - m if e - m >= lo else None
    if d > limits[3]:
        return None
    for s in range(max(lo, e - m - d), e + 1):
        if lev(P, S[s:e]) == d:
            return s
    return None


def item_smem(m, w, d, limits, free=False):
    """The shared-memory bytes fzb_align gives an item (include/fuzzb200.h), 0 for none (no table or no alignment)."""
    S, I, D, L = limits

    def V(layers, b):
        return (6 * layers * (b // 2 + 2) + 15) // 16 * 16

    def T(layers, b):
        return 4 * ((layers * (m + 1) * b + 15) // 16)
    cls = classify(*limits)
    if cls in ("exact", "hamming"):
        return 0
    de = min(d, L) if free else min(d, L, max(m, w))
    if cls == "levenshtein":
        if free:
            return max(V(1, 2 * de + 1) + 4 * de + 2, V(1, de + 1) + T(1, de + 1))
        if abs(w - m) > de:
            return 0
        bw = abs(w - m) + 2 * ((de - abs(w - m)) // 2) + 1
        return V(1, bw) + T(1, bw)
    Ip, Dp = min(I, de), min(D, de)
    return V(Ip + 1, Dp + 1) + T(Ip + 1, Dp + 1)


# ---- brute force -------------------------------------------------------------------------------------------------
def all_alignments(P, T):
    """Every op string aligning P with T."""
    if not P and not T:
        yield ""
        return
    if P and T:
        for rest in all_alignments(P[1:], T[1:]):
            yield ("=" if P[0] == T[0] else "X") + rest
    if P:
        for rest in all_alignments(P[1:], T):
            yield "D" + rest
    if T:
        for rest in all_alignments(P, T[1:]):
            yield "I" + rest


def brute(P, T, limits, d):
    """The rules as a choice among all alignments: the smallest total within the limits and the bound; generic: then
    the fewest insertions; then the canonical one, the walk back from the end that prefers the diagonal, then D, then
    I (the smallest reversed op string with = and X before D before I)."""
    S, I, D, L = limits
    cls = classify(*limits)
    m, w = len(P), len(T)
    key = {"=": 0, "X": 0, "D": 1, "I": 2}
    cands = []
    for ops in all_alignments(P, T):
        x, i, dl = ops.count("X"), ops.count("I"), ops.count("D")
        if cls in ("exact", "hamming"):
            if i or dl or x > (0 if cls == "exact" else min(d, S, L)):
                continue
        else:
            bound = min(d, L, max(m, w))
            if x + i + dl > bound or (cls == "generic" and (x > S or i > I or dl > D)):
                continue
        cands.append((x + i + dl, i if cls == "generic" else 0, [key[c] for c in reversed(ops)], ops))
    if not cands:
        return None
    c = min(cands)
    return c[0], c[3]


LIMITS = [  # (S, I, D, L): every class, with limits that bind
    (BIG, BIG, BIG, 0), (BIG, 0, 0, 2), (1, 0, 0, BIG), (BIG, BIG, BIG, 1), (BIG, BIG, BIG, 3), (2, 2, 2, 2),
    (BIG, 0, 1, 3), (BIG, 1, 0, 3), (0, 1, 1, 2), (1, 1, 1, 3), (3, 0, 2, 3), (2, 2, 0, 4), (0, 3, 3, 6),
    (1, 2, 1, 2),
]


@pytest.mark.parametrize("limits", LIMITS)
def test_restatement_equals_brute_force(limits):
    rng = random.Random(hash(limits) & 0xFFFF)
    cls = classify(*limits)
    for _ in range(150):
        alpha = rng.choice(["AB", "ABC", "ABCD"])
        m = rng.randint(1, 6)
        w = m if cls in ("exact", "hamming") else rng.randint(0, 6)
        P = "".join(rng.choice(alpha) for _ in range(m))
        T = "".join(rng.choice(alpha) for _ in range(w))
        for d in (0, 1, 2, 3, m, 9):
            assert align_anchored(P, T, limits, d) == brute(P, T, limits, d), (P, T, limits, d)


def test_every_pair_of_short_strings_levenshtein():
    """All pairs over {A, B} up to 4 symbols: the restatement's cost is the edit distance and its alignment the
    canonical one."""
    lim = (BIG, BIG, BIG, BIG)
    for m in range(1, 5):
        for w in range(0, 5):
            for P in itertools.product("AB", repeat=m):
                for T in itertools.product("AB", repeat=w):
                    assert align_anchored(P, T, lim, BIG) == brute(P, T, lim, BIG)


def test_tie_rules_and_binding_limits():
    lev_lim = (BIG, BIG, BIG, 2)
    assert align_anchored("A", "AA", lev_lim, 1) == (1, "I=")     # the diagonal last: the I goes first
    assert align_anchored("AA", "A", lev_lim, 1) == (1, "D=")
    assert align_anchored("AB", "BA", lev_lim, 2) == (2, "XX")   # the diagonal before D + I
    assert cigar(align_anchored("ABCDE", "ABDEX", lev_lim, 2)[1]) == "2=1D2=1I"
    # max_insertions = 0 (and so no deletion: the window has the pattern's length) forces substitutions where
    # Levenshtein takes an indel pair
    gen = (3, 0, 1, 3)
    assert classify(*gen) == "generic"
    assert align_anchored("ABCDE", "ABDEX", gen, 3) == (3, "==XXX")
    assert brute("ABCDE", "ABDEX", gen, 3) == (3, "==XXX")
    # max_deletions = 0: a missing pattern symbol has to be paid with substitutions and an insertion elsewhere
    assert align_anchored("ABC", "AC", (2, 1, 0, 3), 3) is None          # w < m needs a deletion
    assert align_anchored("ABCD", "ACDX", (2, 1, 0, 3), 3) == brute("ABCD", "ACDX", (2, 1, 0, 3), 3)
    # the generic final state: the smallest total, then the fewest insertions
    assert align_anchored("AB", "BA", (2, 1, 1, 2), 2) == (2, "XX")
    # the bound: above it there is no alignment
    assert align_anchored("AAAA", "BBBB", (BIG, BIG, BIG, 3), 3) is None
    assert align_anchored("AAAA", "BBBB", (BIG, 0, 0, 3), 3) is None
    assert align_anchored("AAAA", "AAAB", (BIG, BIG, BIG, 0), 0) is None


def test_free_start_equals_brute_force():
    rng = random.Random(11)
    for _ in range(300):
        P = "".join(rng.choice("AB") for _ in range(rng.randint(1, 5)))
        S = "".join(rng.choice("AB") for _ in range(rng.randint(0, 12)))
        lo = rng.randint(0, len(S))
        e = rng.randint(lo, len(S))
        d = min(lev(P, S[s:e]) for s in range(lo, e + 1))  # the nearest distance of P ending at e
        s = free_start(P, S, e, lo, (BIG, BIG, BIG, BIG), d)
        assert s == min(s2 for s2 in range(lo, e + 1) if lev(P, S[s2:e]) == d)
        assert s >= max(lo, e - len(P) - d)
        assert free_start(P, S, e, lo, (BIG, 0, 0, BIG), d) == (e - len(P) if e - len(P) >= lo else None)


def test_item_smem_limits():
    """Every Levenshtein item with d <= m fits, so do the common generic limits, and the largest generic table
    sits where the header says."""
    for m in (1, 64, 65, 255):
        for d in range(0, m + 1, max(1, m // 16)):
            for w in range(max(0, m - d), m + d + 1, max(1, d // 4)):
                assert item_smem(m, w, d, (BIG, BIG, BIG, BIG)) <= 17 * 1024
            assert item_smem(m, 0, d, (BIG, BIG, BIG, BIG), free=True) <= 17 * 1024
        assert item_smem(m, 2 * m, 2 * m, (BIG, BIG, BIG, BIG)) <= 34 * 1024
        for i in range(4):
            for dl in range(4):
                assert item_smem(m, m, 63, (BIG, i, dl, 63)) <= SMEM_MAX
    at, over = generic_at_budget()
    assert item_smem(*at) <= SMEM_MAX < item_smem(*over)


def generic_at_budget():
    """(m, w, d, limits) of a generic item whose table is the largest that fits, and of the one a step above"""
    m, dl = 255, 15
    ins = max(i for i in range(200) if item_smem(m, m, 200, (BIG, i, dl, 200)) <= SMEM_MAX)
    return (m, m, 200, (BIG, ins, dl, 200)), (m, m, 200, (BIG, ins + 1, dl, 200))


def test_cigars_from_op_bytes():
    """The numpy run-length encoding of the op bytes of many items, rows without an alignment left empty."""
    rng = random.Random(3)
    items = ["".join(rng.choice("=XID") for _ in range(rng.randint(1, 30))) for _ in range(200)]
    items[5] = "="
    valid = np.array([rng.random() < 0.8 for _ in items])
    room = [len(x) + rng.randint(0, 4) for x in items]
    offs = np.zeros(len(items) + 1, dtype=np.uint64)
    offs[1:] = np.cumsum(room)
    ops = np.zeros(int(offs[-1]), dtype=np.uint8)
    for x, o in zip(items, offs[:-1].tolist()):
        ops[o:o + len(x)] = np.frombuffer(x.encode(), dtype=np.uint8)
    got = _cigars(ops, offs, [len(x) for x in items], valid)
    assert got == [cigar(x) if v else "" for x, v in zip(items, valid)]
    assert _cigars(ops, offs, [len(x) for x in items], np.zeros(len(items), bool)) == [""] * len(items)
