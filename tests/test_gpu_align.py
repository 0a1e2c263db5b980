"""fzb_align, align_matches and align_in_each (DESIGN.md section 5.17): the edit operations of matches, on the device.
Every alignment is compared exactly with the plain-Python restatement of tests/test_host_align.py (`align_anchored`,
`free_start`), which is checked there against brute force.  `small` keeps the sizes the CPU emulator replays
(tests/test_emu_align.py)."""
import numpy as np
import pytest

from conftest import needs_real_gpu
from fuzzysearch_b200 import (Alignments, DeviceSequence, DeviceSequenceSet, _native as F, align_in_each,
                              align_matches, best_match_in_each, find_near_matches, find_near_matches_in_each,
                              nearest_distance_in_each, nearest_pattern_in_each)
from parity import load_golden
from test_gpu_records import joined, rand
from test_host_align import BIG, align_anchored, classify, cigar, free_start, generic_at_budget, item_smem

pytestmark = pytest.mark.gpu


def norm(subs=None, ins=None, dels=None, l=None):
    from fuzzysearch_b200.search import _normalised_limits
    from fuzzysearch_b200.common import LevenshteinSearchParams
    return _normalised_limits(LevenshteinSearchParams(subs, ins, dels, l))


def expand(c):
    """'2=1X' -> '==X'"""
    out, num = [], ""
    for ch in c:
        if ch.isdigit():
            num += ch
        else:
            out.append(ch * int(num))
            num = ""
    return "".join(out)


def replay(P, T, ops):
    """-> (pattern, window) rebuilt from the ops (a substituted or inserted symbol of the window is taken from T,
    which only checks the op counts and positions; the = pairs are checked to be equal)"""
    i = j = 0
    p, t = [], []
    for op in ops:
        if op in "=X":
            assert (P[i] == T[j]) == (op == "="), (P, T, ops)
            p.append(P[i])
            t.append(T[j])
            i, j = i + 1, j + 1
        elif op == "D":
            p.append(P[i])
            i += 1
        else:
            t.append(T[j])
            j += 1
    return p, t


def check_alignment(P, T, c, limits, dist, exact_cost):
    """Invariants of one alignment, then equality with the restatement."""
    ops = expand(c)
    p, t = replay(P, T, ops)
    assert list(p) == list(P) and list(t) == list(T), (P, T, c)
    n = {k: ops.count(k) for k in "=XID"}
    assert n["="] + n["X"] + n["D"] == len(P) and n["="] + n["X"] + n["I"] == len(T)
    S, I, D, L = limits
    cost = n["X"] + n["I"] + n["D"]
    assert cost <= dist and cost <= L and n["X"] <= S and n["I"] <= I and n["D"] <= D
    if exact_cost:
        assert cost == dist
    want = align_anchored(P, T, limits, dist)
    assert want is not None and cigar(want[1]) == c, (P, T, limits, dist, c, want)
    return cost


def device_align(P, S, ms, limits):
    """Every match aligned through fzb_align directly -> CIGAR or None (cost -1) per match; align_matches returns the
    same list when no match is None and raises ValueError otherwise."""
    from fuzzysearch_b200.search import _cigars
    hs = F.Haystack.from_host(S)
    (_, cost, _, ins, _), ops, oo, _ = hs.align([P], *[[x] for x in limits], [0] * len(ms), [x.start for x in ms],
                                                [x.end for x in ms], [x.dist for x in ms])
    hs.close()
    cig = _cigars(ops, oo, len(P) + ins, cost >= 0)
    return [c if k >= 0 else None for c, k in zip(cig, cost.tolist())]


def check_matches(P, S, ms, kw, limits):
    """-> (Levenshtein matches aligned below their dist, generic matches without an alignment within their dist)"""
    cls = classify(*limits)
    got = device_align(P, S, ms, limits)
    below = unaligned = 0
    for x, c in zip(ms, got):
        if c is None:
            # only the generic search books a substitution, once its substitutions are used up, as an insertion plus
            # a deletion of total cost 1 (generic_search.py): that edit has no alignment within dist
            assert cls == "generic" and align_anchored(P, S[x.start:x.end], limits, x.dist) is None, (P, x)
            unaligned += 1
            continue
        cost = check_alignment(P, S[x.start:x.end], c, limits, x.dist, cls in ("exact", "hamming"))
        below += cls == "levenshtein" and cost < x.dist
    if unaligned:
        with pytest.raises(ValueError):
            align_matches(P, S, ms, **kw)
    else:
        assert align_matches(P, S, ms, **kw) == got
        assert align_matches(P, DeviceSequence(S), ms, **kw) == got
    return below, unaligned


def planted(rng, alphabet, n, P, k, edits):
    """A text of n symbols with k copies of P carrying up to `edits` random edits each"""
    S = bytearray(rand(rng, alphabet, n))
    alpha = np.frombuffer(alphabet, dtype=np.uint8)
    for at in rng.integers(0, n - 2 * len(P), size=k):
        v = bytearray(P)
        for _ in range(int(rng.integers(0, edits + 1))):
            kind, x = int(rng.integers(0, 3)), int(rng.integers(0, len(v)))
            if kind == 0:
                v[x] = int(alpha[rng.integers(0, len(alpha))])
            elif kind == 1 and len(v) > 1:
                del v[x]
            else:
                v.insert(x, int(alpha[rng.integers(0, len(alpha))]))
        S[at:at + len(v)] = v
    return bytes(S)


# (limits as find_near_matches takes them, pattern length): every class and both routes of the searches
CASES = [
    (dict(max_l_dist=0), 12),                                                          # exact
    (dict(max_substitutions=2, max_insertions=0, max_deletions=0), 20),                # substitutions only
    (dict(max_l_dist=2), 30),                                                          # Levenshtein, n-grams
    (dict(max_l_dist=3), 8),                                                           # Levenshtein, LP
    (dict(max_substitutions=2, max_insertions=1, max_deletions=1, max_l_dist=2), 30),  # generic, n-grams
    (dict(max_substitutions=1, max_insertions=2, max_deletions=0, max_l_dist=3), 9),   # generic, LP
    (dict(max_substitutions=0, max_insertions=1, max_deletions=2, max_l_dist=2), 12),
]


@pytest.mark.parametrize("alphabet", [b"ACGT", bytes(range(32, 127))])
def test_every_match_of_every_class(cuda_device, alphabet, small=False):
    rng = np.random.default_rng(len(alphabet))
    for kw, m in CASES:
        limits = norm(kw.get("max_substitutions"), kw.get("max_insertions"), kw.get("max_deletions"),
                      kw.get("max_l_dist"))
        cls = classify(*limits)
        P = rand(rng, alphabet, m)
        S = planted(rng, alphabet, 20000 if small else 200000, P, 30 if small else 300,
                    0 if cls == "exact" else 3)
        ms = find_near_matches(P, S, **kw)
        assert ms, kw
        below, unaligned = check_matches(P, S, ms, kw, limits)
        print("%s: %d matches, %d aligned below their dist, %d without an alignment within it" %
              (kw, len(ms), below, unaligned))


def test_golden_fuzz_matches(cuda_device, stride=1):
    """Every match of the stored find_near_matches calls of the reference (tests/golden/ref_fuzz.json)."""
    counts = {}
    for rec in [r for r in load_golden("ref_fuzz.json") if r["fn"] == "find_near_matches" and "exc" not in r][::stride]:
        a = rec["args"]
        P, S = bytes.fromhex(a[0]), bytes.fromhex(a[1])
        ms = find_near_matches(P, S, *a[2:6])
        if not ms:
            continue
        limits = norm(*a[2:6])
        kw = dict(zip(("max_substitutions", "max_insertions", "max_deletions", "max_l_dist"), a[2:6]))
        c = counts.setdefault(classify(*limits), [0, 0, 0])
        below, unaligned = check_matches(P, S, ms, kw, limits)
        c[0] += len(ms)
        c[1] += below
        c[2] += unaligned
    print("golden matches per class: [matches, aligned below their dist, without an alignment within it]", counts)


def test_wide_symbols_and_items(cuda_device):
    P, S = "naïve ☃ café", "xx naive ☃ cafe yy naïve ☃ café"
    ms = find_near_matches(P, S, max_l_dist=2)
    cig = align_matches(P, S, ms, max_l_dist=2)
    for x, c in zip(ms, cig):
        check_alignment(P, S[x.start:x.end], c, norm(l=2), x.dist, False)
    items = [1, 2, 3, 4, 5]
    ms = find_near_matches(items, [9, 1, 2, 7, 4, 5, 9], max_l_dist=1)
    assert align_matches(items, [9, 1, 2, 7, 4, 5, 9], ms, max_l_dist=1) == ["2=1X2="]


def check_rows(P_list, seqs, rows, al, limits_of, nearest):
    """Each row of `al` equals the restatement on its read: the smallest start for nearest rows, cost == dist."""
    for r in range(len(seqs)):
        pi = int(rows.pattern[r]) if hasattr(rows, "pattern") else (0 if rows.dist[r] >= 0 else -1)
        if pi < 0:
            assert al[r] is None and al.cigar[r] == "" and al.dist[r] == -1
            continue
        P, S, lim = P_list[pi], seqs[r], limits_of(pi)
        e = int(rows.end[r])
        if nearest:
            s = free_start(P, S, e, 0, lim, int(rows.dist[r]))
            assert al.dist[r] == rows.dist[r]
        else:
            s = int(rows.start[r])
        assert (al.start[r], al.end[r]) == (s, e), r
        check_alignment(P, S[s:e], al.cigar[r], lim, int(rows.dist[r]), nearest or classify(*lim) == "hamming")
        assert al.substitutions[r] + al.insertions[r] + al.deletions[r] == al.dist[r]


def test_align_in_each_rows(cuda_device, small=False):
    rng = np.random.default_rng(21)
    n = 3000 if small else 100000
    bcs = [rand(rng, b"ACGT", 12) for _ in range(8)]
    seqs = []
    for r in range(n):
        t = bytearray(rand(rng, b"ACGT", int(rng.integers(0, 60))))
        if r % 3 and len(t) > 14:
            at = int(rng.integers(0, len(t) - 13))
            b = bytearray(bcs[r % 8])
            b[int(rng.integers(0, 12))] = ord("ACGT"[r % 4])
            if r % 5 == 0:
                del b[3]
            t[at:at + len(b)] = b
        seqs.append(bytes(t))
    sample = rng.choice(n, size=300 if small else 1500, replace=False)
    resident = DeviceSequenceSet(seqs)
    kw = dict(max_substitutions=2, max_insertions=1, max_deletions=1)
    best = best_match_in_each(bcs, seqs, 2, **kw)
    al = align_in_each(bcs, seqs, best, 2, **kw)
    assert isinstance(al, Alignments)
    al2 = align_in_each(bcs, resident, best, 2, **kw)
    for c in ("start", "end", "dist", "substitutions", "insertions", "deletions"):
        assert (getattr(al, c) == getattr(al2, c)).all()
    assert al.cigar == al2.cigar
    lim = norm(2, 1, 1, 2)
    check_rows(bcs, [seqs[r] for r in sample], _Sub(best, sample), _Sub(al, sample), lambda i: lim, False)
    for r in sample[:100]:
        if best.pattern[r] >= 0:
            one = align_matches(bcs[best.pattern[r]], seqs[r], [best[r][1]], 2, 1, 1, 2)
            assert one == [al.cigar[r]]
    for subs_only in (False, True):
        lim = norm(BIG, 0, 0, BIG) if subs_only else norm(BIG, BIG, BIG, BIG)
        near = nearest_pattern_in_each(bcs, resident, substitutions_only=subs_only)
        al = align_in_each(bcs, resident, near, substitutions_only=subs_only)
        assert ((al.dist == near.dist) | (near.pattern < 0)).all()
        assert (al.end == np.where(near.pattern >= 0, near.end, -1)).all()
        check_rows(bcs, [seqs[r] for r in sample], _Sub(near, sample), _Sub(al, sample), lambda i: lim, True)
        one = nearest_distance_in_each(bcs[3], seqs, substitutions_only=subs_only)
        al = align_in_each(bcs[3], seqs, one, substitutions_only=subs_only)
        assert ((al.dist == one.dist) | (one.dist < 0)).all()
        check_rows([bcs[3]], [seqs[r] for r in sample], _Sub(one, sample), _Sub(al, sample), lambda i: lim, True)
    resident.close()


class _Sub(object):
    """The rows `idx` of a result object (numpy columns by attribute)"""

    def __init__(self, obj, idx):
        self._o, self._i = obj, idx

    def __getattr__(self, name):
        v = getattr(self._o, name)
        return [v[i] for i in self._i] if isinstance(v, list) else np.asarray(v)[self._i]

    def __getitem__(self, r):
        return self._o[int(self._i[r])]


def test_edges(cuda_device):
    rng = np.random.default_rng(4)
    lev = norm(BIG, BIG, BIG, BIG)
    for m in (1, 64, 65, 255):
        P = rand(rng, b"ACGT", m)
        for d in sorted({0, 1, m // 2, m}):
            # anchored windows of every length the bound allows, and free starts at d = the nearest distance
            recs = [rand(rng, b"ACGT", int(x)) for x in rng.integers(0, 3 * m, size=12)] + [b"", P, P[: m // 2]]
            buf, off = joined(recs)
            hs = F.Haystack.from_host(buf)
            hs.set_records(off)
            items = []
            for r, t in enumerate(recs):
                for w in {max(0, m - d), m, min(len(t), m + d), len(t)}:
                    if w <= len(t):
                        s = int(rng.integers(0, len(t) - w + 1))
                        items.append((int(off[r]) + s, int(off[r]) + s + w, t[s:s + w], d, r))
            (start, cost, x, ins, dels), ops, oo, st = hs.align([P], [lev[0]], [lev[1]], [lev[2]], [lev[3]],
                                                                [0] * len(items), [i[0] for i in items],
                                                                [i[1] for i in items], [i[3] for i in items])
            assert st["route"] == "alignment"
            for k, (s, e, T, dd, r) in enumerate(items):
                want = align_anchored(P, T, lev, dd)
                if want is None:
                    assert cost[k] == start[k] == -1, (m, d, k)
                else:
                    got = bytes(ops[int(oo[k]):int(oo[k]) + m + int(ins[k])]).decode()
                    assert (int(cost[k]), got) == want and start[k] == s, (m, d, k)
                    assert int(x[k]) + int(ins[k]) + int(dels[k]) == cost[k]
            # free starts: the nearest distance of each record, clipped at the record's first symbol
            near = nearest_distance_in_each(P, recs)
            al = align_in_each(P, recs, near)
            for r, t in enumerate(recs):
                s = free_start(P, t, int(near.end[r]), 0, lev, int(near.dist[r]))
                assert (al.start[r], al.dist[r]) == (s, near.dist[r]), (m, r)
            hs.close()


def test_rows_without_matches_and_empty_records(cuda_device):
    seqs = [b"", b"ACGT", b"", b"TTTTTTTT"]
    best = best_match_in_each([b"GGGGG"], seqs, 1)
    al = align_in_each([b"GGGGG"], seqs, best, 1)
    assert (al.start == -1).all() and al.cigar == [""] * 4 and [al[r] for r in range(4)] == [None] * 4
    near = nearest_pattern_in_each([b"ACGTA", b"GG"], seqs, substitutions_only=True)
    al = align_in_each([b"ACGTA", b"GG"], seqs, near, substitutions_only=True)
    assert al[0] is None and al[2] is None and al[1] == (1, 3, "1X1=") and al[3] == (0, 2, "2X")
    near = nearest_distance_in_each(b"ACG", seqs)
    al = align_in_each(b"ACG", seqs, near)
    assert al[0] == (0, 0, "3D") and al[1] == (0, 3, "3=") and al[3] == (0, 0, "3D")


def test_generic_table_budget(cuda_device):
    """A generic item whose table is exactly the largest that fits runs; one a step above is refused."""
    (m, w, d, lim_at), (_, _, _, lim_over) = generic_at_budget()
    rng = np.random.default_rng(8)
    P = rand(rng, b"ACGT", m)
    T = bytearray(P)
    T[7] ^= 2
    hs = F.Haystack.from_host(bytes(T))
    (start, cost, x, ins, dels), ops, oo, _ = hs.align([P], [lim_at[0]], [lim_at[1]], [lim_at[2]], [lim_at[3]], [0],
                                                       [0], [m], [d])
    assert (int(start[0]), int(cost[0]), int(x[0])) == (0, 1, 1)
    assert item_smem(m, w, d, lim_at) <= 64 * 1024 < item_smem(m, w, d, lim_over)
    with pytest.raises(F.UnsupportedError):
        hs.align([P], [lim_over[0]], [lim_over[1]], [lim_over[2]], [lim_over[3]], [0], [0], [m], [d])
    hs.close()


def test_refusals_leave_the_handle_usable(cuda_device):
    P = b"GATTACA"
    recs = [b"xxGATTACAxx", b"GATACA", b"TTTT"]
    buf, off = joined(recs)
    hs = F.Haystack.from_host(buf)
    hs.set_records(off)
    lev, ham, ex, gen = norm(l=1), norm(1, 0, 0), norm(l=0), norm(1, 1, 0, 2)

    def call(lim, s, e, d=1, pat=0, pats=(P,)):
        return hs.align(list(pats), [lim[0]], [lim[1]], [lim[2]], [lim[3]], [pat], [s], [e], [d])

    good = call(lev, 2, 9)[0]
    assert good[1][0] == 0
    bad = [
        (lev, 2, len(buf) + 1),       # outside the buffer
        (lev, 10, 13),                # crosses a record edge (record 0 ends at 11)
        (lev, 9, 5),                  # start > end
        (ex, -1, 9),                  # free start on an exact pattern
        (gen, -1, 9),                 # ... and on a generic one
        (ham, 2, 8),                  # a substitutions-only window shorter than m
        (ex, 2, 10),                  # an exact window longer than m
    ]
    for lim, s, e in bad:
        with pytest.raises(ValueError):
            call(lim, s, e)
        assert find_near_matches_in_each(P, DeviceSequenceSet(recs), max_l_dist=1)[0][0].start == 2
        assert [r.tolist() for r in hs.align([P], [lev[0]], [lev[1]], [lev[2]], [lev[3]], [0], [2], [9], [1])[0]] == \
            [r.tolist() for r in good]
    with pytest.raises(ValueError):
        call(lev, 2, 9, pat=1)        # unknown pattern index
    res = hs.search_levenshtein(P, 1)
    assert res.triples()[0][:2] == (2, 9)
    with pytest.raises(F.UnsupportedError):
        hs.align([P], [lev[0]], [lev[1]], [lev[2]], [lev[3]], [0], [2], [9], [1], flags=F.F_TINY_LIST)
    assert res.triples()[0][:2] == (2, 9)  # the pending result of the search is untouched
    res.close()
    with pytest.raises(ValueError):
        align_matches(P, b"xxGATGACAxx", find_near_matches(P, b"xxGATGACAxx", max_l_dist=1), max_l_dist=0)
    with pytest.raises((ValueError, TypeError)):  # validated as find_near_matches validates, before any upload
        align_matches(P, b"xxGATTACAxx", [], max_l_dist=-1)
    hs.close()


def test_item_past_2_32(cuda_device):
    """Items whose windows sit above 2^32 in buffer coordinates."""
    needs_real_gpu("a 4 GiB sequence")
    n = (1 << 32) + (1 << 20)
    hs = F.Haystack.alloc(n)
    hs.fill_synthetic(b"ACGT", 5)
    P = b"GATTACAGATTACAGATTACA"
    at = (1 << 32) - 9
    hs.write(at, P[:10] + b"N" + P[11:])
    hs.write(n - len(P), P)
    lev = norm(l=2)
    (start, cost, x, ins, dels), ops, oo, _ = hs.align([P], [lev[0]], [lev[1]], [lev[2]], [lev[3]], [0, 0, 0],
                                                       [at, n - len(P), -1], [at + len(P), n, n], [1, 0, 0])
    assert start.tolist() == [at, n - len(P), n - len(P)] and cost.tolist() == [1, 0, 0]
    assert bytes(ops[int(oo[0]):int(oo[0]) + len(P)]) == b"=" * 10 + b"X" + b"=" * 10
    hs.close()
