"""The single-pattern routes built on a candidate NFA, at their limits: the Levenshtein LP route (streaming
k_lp_scan + k_lp_verify, and the k_lev_lp tile kernel) and the generic route (k_generic_lp over the whole sequence,
k_verify_generic on the n-gram windows).  Every search is compared with the oracle, raw multiset and final list.

Which path a search took is read from stats()["n_launches"].  One attempt of the streaming LP search is 3 launches
(k_lp_scan, k_lp_verify, k_post), one of the tile kernel 2 (k_lev_lp or k_generic_lp, k_post), one of the generic
n-gram route 3 (filter, k_verify_generic, k_post).  A start with more live candidates than the per-thread lists hold
repeats the attempt with lists 8 times longer (256, 2 048, 16 384 entries), and a raw stream longer than the output
buffer repeats it with a larger buffer, which the handle keeps."""
import numpy as np
import pytest

import oracle
from corpus import ASCII, DNA, make_corpus, mutate
from fuzzysearch_b200 import _native as F
from fuzzysearch_b200 import find_near_matches
from parity import tup

pytestmark = pytest.mark.gpu

LP, LP_TILE = F.F_FORCE_LP, F.F_FORCE_LP | F.F_FORCE_DENSE
STREAM_ATTEMPT, TILE_ATTEMPT, NGRAM_ATTEMPT = 3, 2, 3   # launches per attempt
CAND_CAP = 16384                                        # longest candidate list of one start (api.cu: kLpMaxCap)
LOOK_AHEAD_WIN = 48                                     # widest m + k of the streaming form (kLpsMaxWin)
SHIFTS = (1 << 32, (1 << 35) - 4096, (1 << 40) + 16 * 12345, 1 << 44)


# ---- restatements of the device simulations that count list lengths (lp_kernels.cuh) --------------------------
def lev_lp_peak(pat, hay, k, start, stop=CAND_CAP + 1):
    """Longest candidate list sim_lev_lp builds for `start` (stops counting above `stop`)."""
    m, n = len(pat), len(hay)
    j0 = next((j for j in range(min(k, m - 1) + 1) if pat[j] == hay[start]), -1)
    if j0 < 0 or j0 + 1 == m:
        return 0
    cands, peak = [(j0 + 1, j0)], 1
    for i in range(start + 1, n):
        c, nxt = hay[i], []
        for j, d in cands:
            if pat[j] == c:
                if j + 1 != m:
                    nxt.append((j + 1, d))
            elif d < k:
                nxt.append((j, d + 1))
                if i + 1 < n and j + 1 < m:
                    nxt.append((j + 1, d + 1))
                for t in range(1, k - d + 1):
                    if j + t == m:
                        break
                    if pat[j + t] == c:
                        if j + t + 1 != m:
                            nxt.append((j + 1 + t, d + t))
                        break
        peak = max(peak, len(nxt))
        if not nxt or peak > stop:
            break
        cands = nxt
    return peak


def generic_peak(pat, hay, subs, ins, dels, max_l, start, stop=CAND_CAP + 1):
    """Longest candidate list sim_generic builds for `start` over the whole sequence."""
    m = len(pat)
    cands, peak = [(0, 0, 0, 0, 0)], 1
    for i in range(start, len(hay)):
        c, nxt = hay[i], []
        for j, l, ns, ni, nd in cands:
            if c == pat[j]:
                if j + 1 != m:
                    nxt.append((j + 1, l, ns, ni, nd))
            elif l < max_l:
                if ni < ins:
                    nxt.append((j, l + 1, ns, ni + 1, nd))
                if j + 1 < m:
                    if ns < subs:
                        nxt.append((j + 1, l + 1, ns + 1, ni, nd))
                    elif nd < dels and ni < ins:
                        nxt.append((j + 1, l + 1, ns, ni + 1, nd + 1))
                for t in range(1, min(dels - nd, max_l - l) + 1):
                    if j + t == m:
                        break
                    if pat[j + t] == c:
                        if j + t + 1 != m:
                            nxt.append((j + 1 + t, l + t, ns, ni, nd + t))
                        break
        peak = max(peak, len(nxt))
        if not nxt or peak > stop:
            break
        cands = nxt
    return peak


# ---- helpers ---------------------------------------------------------------------------------------------------
def check(res, cpu):
    assert sorted(res.triples(F.RAW)) == sorted(tup(cpu))
    assert res.triples(F.FINAL) == tup(oracle.consolidate(cpu))


def launches(res):
    return res.stats()["n_launches"]


def settled(hs, search, cpu):
    """Runs `search` twice on the handle hs, checks both against cpu -> the second run's launches, which count only
    the candidate attempts (the first run has grown the output buffer if the raw stream needed it)."""
    first = search()
    check(first, cpu)
    first.close()
    again = search()
    check(again, cpu)
    assert again.stats()["route"] == "lp" or again.stats()["route"].startswith("generic")
    n = launches(again)
    again.close()
    return n


def plant_subs(rng, hay, pat, nsubs, pos, alphabet):
    """pat with nsubs substitutions (never the first character: the LP route opens a candidate on it) at pos."""
    v = bytearray(pat)
    for j in rng.choice(np.arange(1, len(pat)), size=min(nsubs, len(pat) - 1), replace=False):
        v[j] = next(c for c in alphabet if c != pat[j])
    hay[pos:pos + len(v)] = np.frombuffer(bytes(v), dtype=np.uint8)


def lev_input(alphabet, n, m, k, seed):
    """make_corpus's plants (up to k + 1 edits, clusters, both global ends), plus copies with exactly k substitutions
    and a prefix of m - k characters at the very end (accepted there with distance exactly k)."""
    pat, hay, _ = make_corpus(seed, n, alphabet, m, 16, k + 1)
    rng = np.random.default_rng(seed)
    for pos in range(2 * m, n - 3 * m, max(n // 8, 3 * m)):
        plant_subs(rng, hay, pat, k, pos, alphabet)
    hay[n - (m - k):] = np.frombuffer(pat[:m - k], dtype=np.uint8)
    return pat, hay


# ---- k_lp_verify and the streaming window --------------------------------------------------------------------
@pytest.mark.parametrize("alphabet,n,m,k,want", [
    # (launches plain, with the tile kernel forced): 3 / 2 per attempt, k >= 8 needs more than 256 candidates
    (ASCII, 20000, 14, 4, (3, 2)),    # lp_nfa_any<4> at its largest k
    (ASCII, 20000, 14, 5, (3, 2)),    # lp_nfa_any<8> at its smallest k
    (ASCII, 20000, 29, 4, (3, 2)),    # <4> with the top bits of the 32-bit masks
    (ASCII, 20000, 31, 8, (6, 4)),    # <8> at its largest k, m = 31: bit 30 of the masks
    (ASCII, 20000, 27, 9, (6, 4)),    # k = 9: the literal simulation only
    (ASCII, 20000, 32, 8, (6, 4)),    # m = 32: the literal simulation only
    (ASCII, 20000, 36, 11, (9, 6)),   # window 47
    (ASCII, 20000, 36, 12, (9, 6)),   # window 48: the whole 64-bit look-ahead
    (ASCII, 20000, 37, 12, (6, 6)),   # window 49: the tile kernel
    (ASCII, 20000, 38, 12, (6, 6)),   # window 50
    (DNA, 3000, 12, 4, (3, 2)),
    (DNA, 3000, 12, 5, (3, 2)),
    (DNA, 3000, 26, 8, (6, 4)),
    (DNA, 3000, 31, 6, (3, 2)),
    (DNA, 3000, 32, 6, (3, 2)),
    (DNA, 3000, 40, 7, (6, 4)),       # window 47
    (DNA, 3000, 41, 7, (6, 4)),       # window 48
    (DNA, 3000, 42, 7, (4, 4)),       # window 49
    (DNA, 3000, 43, 7, (4, 4)),       # window 50
])
def test_lp_verify_and_window_boundaries(cuda_device, alphabet, n, m, k, want):
    """Every mode of k_lp_verify (lp_nfa_any<4> for k <= 4, <8> for k <= 8, the literal simulation for m > 31 or
    k > 8) and the streaming form up to window m + k = 48; above it the tile kernel takes the search.  The plain
    search and the tile kernel must both give the oracle's multiset."""
    pat, hay = lev_input(alphabet, n, m, k, 100 * m + k)
    cpu = oracle.levenshtein_lp_raw(pat, hay, k)
    assert len(cpu) >= 16
    hs = F.Haystack.from_host(hay)
    plain, tile = settled(hs, lambda: hs.search_levenshtein(pat, k, LP), cpu), \
        settled(hs, lambda: hs.search_levenshtein(pat, k, LP_TILE), cpu)
    assert (plain, tile) == want
    if m + k <= LOOK_AHEAD_WIN:
        assert plain // STREAM_ATTEMPT == tile // TILE_ATTEMPT and plain % STREAM_ATTEMPT == 0
    else:
        assert plain == tile
    hs.close()


@pytest.mark.parametrize("k,attempts", [(11, 2), (12, 3)])
def test_lp_scan_look_ahead(cuda_device, k, attempts):
    """k_lp_scan counts the pattern's characters in the window m + k (47, 48) from the masks of its own lane and the
    next three.  Copies whose count is exactly m - k, or which reach the window's last bytes, sit at every offset
    within a lane and a warp; the text has no character of the pattern, so each count is tight."""
    rng = np.random.default_rng(47 + k)
    m = 36
    letters = np.frombuffer(ASCII[33:59] + ASCII[65:91], dtype=np.uint8)   # A-Z, a-z
    pat = bytes(rng.choice(letters, size=m))
    other = np.array([c for c in ASCII if c not in pat], dtype=np.uint8)
    n = 97 * 80 + 200
    hay = other[rng.integers(0, len(other), size=n)].copy()
    junk = bytes(other[:k])
    starts = []
    for q in range(80):  # 97 = 1 (mod 16): every offset within a lane, and varying offsets within a warp
        pos = 50 + 97 * q
        v = pat[:1] + junk + pat[k + 1:] if q % 2 else pat[:1] + junk + pat[1:]   # k substitutions / insertions
        hay[pos:pos + len(v)] = np.frombuffer(v, dtype=np.uint8)
        starts.append(pos)
    cpu = oracle.levenshtein_lp_raw(pat, hay, k)
    assert {s for s, _, _ in tup(cpu)} >= set(starts)
    hs = F.Haystack.from_host(hay)
    assert settled(hs, lambda: hs.search_levenshtein(pat, k, LP), cpu) == attempts * STREAM_ATTEMPT
    assert settled(hs, lambda: hs.search_levenshtein(pat, k, LP_TILE), cpu) == attempts * TILE_ATTEMPT
    hs.close()


def test_lp_survivor_list_overflow(cuda_device):
    """FZB_F_TINY_LIST caps the survivor list at 1 024 starts; on DNA most starts survive k_lp_scan, the list
    overflows, k_lp_verify leaves it and the tile kernel repeats the search.  A normal search on the same handle
    streams again."""
    pat, hay = lev_input(DNA, 6000, 12, 4, 6000)
    cpu = oracle.levenshtein_lp_raw(pat, hay, 4)
    hs = F.Haystack.from_host(hay)
    tiny = hs.search_levenshtein(pat, 4, LP | F.F_TINY_LIST)
    assert launches(tiny) == STREAM_ATTEMPT + TILE_ATTEMPT
    check(tiny, cpu)
    normal = hs.search_levenshtein(pat, 4, LP)
    assert launches(normal) == STREAM_ATTEMPT
    check(normal, cpu)
    tiny.close()
    normal.close()
    hs.close()


# ---- candidate lists ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind,n,m,limits,flags,seed,peak,attempts", [
    ("lev", 300, 16, 7, LP, 2, (256, 2048), 2),
    ("lev", 300, 16, 7, LP_TILE, 2, (256, 2048), 2),
    ("lev", 300, 24, 11, LP, 2, (2048, CAND_CAP), 3),
    ("lev", 300, 24, 11, LP_TILE, 2, (2048, CAND_CAP), 3),
    ("generic", 200, 16, (4, 4, 4, 8), LP, 1, (256, 2048), 2),
    ("generic", 200, 20, (5, 5, 5, 10), LP, 1, (2048, CAND_CAP), 3),
    ("generic", 300, 36, (3, 6, 3, 8), 0, 0, None, 2),       # n-gram route
    ("generic", 300, 36, (4, 6, 4, 10), 0, 0, None, 3),
])
def test_candidate_list_growth(cuda_device, kind, n, m, limits, flags, seed, peak, attempts):
    """Starts with more live candidates than 256, and than 2 048: the search repeats with longer lists.  `peak`
    bounds the longest list of the busiest start (restated on the host).  Each search runs twice on one handle: the
    second run's output buffer is already large enough, so its launches count only the candidate attempts."""
    k = limits if kind == "lev" else limits[3]
    pat, hay, _ = make_corpus(seed, n, DNA, m, 4, k + 1)
    hb = hay.tobytes()
    if kind == "lev":
        cpu = oracle.levenshtein_lp_raw(pat, hay, k)
        top = max(lev_lp_peak(pat, hb, k, s) for s in range(n))
        search = lambda hs: hs.search_levenshtein(pat, k, flags)  # noqa: E731
        per = TILE_ATTEMPT if flags & F.F_FORCE_DENSE else STREAM_ATTEMPT
    elif flags & F.F_FORCE_LP:
        cpu = oracle.generic_lp_raw(pat, hay, *limits)
        top = max(generic_peak(pat, hb, *limits, s) for s in range(n))
        search = lambda hs: hs.search_generic(pat, *limits, flags=flags)  # noqa: E731
        per = TILE_ATTEMPT
    else:
        cpu = oracle.generic_ngrams_raw(pat, hay, *limits)
        search = lambda hs: hs.search_generic(pat, *limits, flags=flags)  # noqa: E731
        per = NGRAM_ATTEMPT
    if peak is not None:
        assert peak[0] < top <= peak[1], top
    hs = F.Haystack.from_host(hay)
    assert settled(hs, lambda: search(hs), cpu) == attempts * per
    hs.close()


def test_candidate_limit(cuda_device):
    """A start with more than 16 384 live candidates fails the search with UnsupportedError naming that limit (the
    reference answers these inputs); the handle stays usable."""
    cases = [("lev", 200, 30, 14, 0), ("generic", 200, 45, (14, 14, 14, 14), 0)]
    for kind, n, m, limits, seed in cases:
        k = limits if kind == "lev" else limits[3]
        pat, hay, _ = make_corpus(seed, n, DNA, m, 4, k + 1)
        hb = hay.tobytes()
        if kind == "lev":
            assert len(oracle.levenshtein_lp_raw(pat, hay, k)) > 0
            assert max(lev_lp_peak(pat, hb, k, s) for s in range(n)) > CAND_CAP
        else:
            assert len(oracle.generic_lp_raw(pat, hay, *limits)) > 0
            assert max(generic_peak(pat, hb, *limits, s) for s in range(n)) > CAND_CAP
        hs = F.Haystack.from_host(hay)
        with pytest.raises(F.UnsupportedError, match="more than 16384 live candidates for one start"):
            if kind == "lev":
                hs.search_levenshtein(pat, k, LP)
            else:
                hs.search_generic(pat, *limits, flags=LP)
        small = pat[:8]
        res = hs.search_levenshtein(small, 3, LP)
        check(res, oracle.levenshtein_lp_raw(small, hay, 3))
        res.close()
        res = hs.search_generic(small, 1, 1, 1, 2, LP)
        check(res, oracle.generic_lp_raw(small, hay, 1, 1, 1, 2))
        res.close()
        hs.close()


# ---- generic route: 6-bit counters, the lowering rule, the n-gram windows ------------------------------------------
def plant_generic(rng, hay, pat, limits, at):
    """Copies that spend a whole limit: max_subs substitutions, max_ins inserted characters, and (max_dels) a prefix
    of m - max_dels characters at the very end (a match there needs exactly max_dels deletions)."""
    subs, ins, dels, _ = limits
    n, m = len(hay), len(pat)
    if subs:
        plant_subs(rng, hay, pat, min(subs, m - 1), at[0], ASCII)
    if ins:
        v = bytearray(pat)
        for _ in range(ins):
            v.insert(int(rng.integers(1, len(v))), int(rng.choice(np.frombuffer(ASCII, dtype=np.uint8))))
        hay[at[1]:at[1] + len(v)] = np.frombuffer(bytes(v), dtype=np.uint8)
    if dels and dels < m:
        hay[n - (m - dels):] = np.frombuffer(pat[:m - dels], dtype=np.uint8)


@pytest.mark.parametrize("m,limits,flags,route", [
    (70, (63, 0, 0, 63), LP, "generic-lp"),
    (40, (0, 63, 0, 63), LP, "generic-lp"),
    (100, (0, 0, 63, 63), LP, "generic-lp"),
    (255, (63, 0, 0, 63), 0, "generic-ngrams"),   # L = 3
    (200, (0, 63, 0, 63), 0, "generic-ngrams"),
    (255, (0, 0, 63, 63), 0, "generic-ngrams"),
    (40, (1, 40, 0, 63), LP, "generic-lp"),       # mixed, 63 after the LP route's lowering (min(63, 40 + 40))
])
def test_generic_counters_at_63(cuda_device, m, limits, flags, route):
    """sim_generic packs each candidate's counters into 6 bits: one of them at 63, the others small (the candidate
    lists stay short), with copies that spend the whole limit."""
    n = 4000
    pat, hay, _ = make_corpus(m + sum(limits), n, ASCII, m, 8, 11)
    rng = np.random.default_rng(m)
    plant_generic(rng, hay, pat, limits, (n // 3, 2 * n // 3))
    lp = bool(flags & F.F_FORCE_LP)
    cpu = oracle.generic_lp_raw(pat, hay, *limits) if lp else oracle.generic_ngrams_raw(pat, hay, *limits)
    assert max(d for _, _, d in tup(cpu)) > 31
    hs = F.Haystack.from_host(hay)
    res = hs.search_generic(pat, *limits, flags=flags)
    assert res.stats()["route"] == route
    check(res, cpu)
    res.close()
    hs.close()


def test_generic_lowering_rule(cuda_device):
    """On the LP route max_l_dist is lowered to m + max_insertions (no candidate can spend more); a lowered total of
    63 runs, 64 does not.  The same through find_near_matches, with max_l_dist=None too (the sum of the limits)."""
    n = 3000
    pat, hay, _ = make_corpus(40, n, ASCII, 40, 8, 11)
    rng = np.random.default_rng(40)
    plant_generic(rng, hay, pat, (0, 23, 0, 100), (n // 3, n // 2))
    hs = F.Haystack.from_host(hay)
    res = hs.search_generic(pat, 0, 23, 0, 100)           # 100 -> 63
    assert res.stats()["route"] == "generic-lp"
    check(res, oracle.generic_lp_raw(pat, hay, 0, 23, 0, 100))
    res.close()
    with pytest.raises(F.UnsupportedError, match="max_l_dist > 63"):
        hs.search_generic(pat, 0, 24, 0, 100)               # 100 -> 64
    hs.close()
    t = lambda ms: [(x.start, x.end, x.dist) for x in ms]  # noqa: E731
    h = hay.tobytes()
    # (find_near_matches first lowers max_l_dist to the sum of the per-operation limits, as the reference does)
    for kw in (dict(max_substitutions=0, max_insertions=24, max_deletions=0, max_l_dist=100),   # -> 24
               dict(max_substitutions=0, max_insertions=63, max_deletions=0),                   # None -> 63
               dict(max_substitutions=0, max_insertions=0, max_deletions=100)):                 # None -> 100 -> 40
        assert t(find_near_matches(pat, h, **kw)) == oracle.find_near_matches(pat, h, **kw), kw
    with pytest.raises(F.UnsupportedError, match="max_l_dist > 63"):
        find_near_matches(pat, h, max_substitutions=0, max_insertions=64, max_deletions=0)    # None -> 64
    long_pat = pat + pat[:30]                                                        # m = 70
    hay[n - 6:] = np.frombuffer(long_pat[:6], dtype=np.uint8)
    h = hay.tobytes()
    kw = dict(max_substitutions=0, max_insertions=0, max_deletions=63)
    assert t(find_near_matches(long_pat, h, **kw)) == oracle.find_near_matches(long_pat, h, **kw)
    with pytest.raises(F.UnsupportedError, match="max_l_dist > 63"):
        find_near_matches(long_pat, h, max_substitutions=0, max_insertions=0, max_deletions=64)  # None -> 64


@pytest.mark.parametrize("limits", [(2, 2, 2, 4), (1, 3, 2, 5), (0, 0, 5, 5)])
def test_generic_ngram_windows_at_global_ends(cuda_device, limits):
    """n-gram hits within m + k of position 0 and of N: the window is clipped there, and its end acts as the end of
    input (a candidate that runs into it may still accept with deletions)."""
    m, k, n = 30, limits[3], 3000
    pat, hay, _ = make_corpus(k, n, ASCII, m, 8, k + 1)
    rng = np.random.default_rng(k)
    tail = pat[:m - limits[2]]  # accepted at N only with every deletion spent
    hay[n - len(tail):] = np.frombuffer(tail, dtype=np.uint8)
    for pos in (1, n - len(tail) - m - 2):  # windows clipped at 0 and at N
        v = mutate(rng, pat, ASCII, 1) if limits[1] and limits[2] else pat
        hay[pos:pos + len(v)] = np.frombuffer(v, dtype=np.uint8)
    cpu = oracle.generic_ngrams_raw(pat, hay, *limits)
    assert min(s for s, _, _ in tup(cpu)) <= k and max(e for _, e, _ in tup(cpu)) == n
    hs = F.Haystack.from_host(hay)
    for flags in (0, F.F_FORCE_DENSE):
        res = hs.search_generic(pat, *limits, flags=flags)
        assert res.stats()["route"] == "generic-ngrams"
        check(res, cpu)
        res.close()
    hs.close()


# ---- shards --------------------------------------------------------------------------------------------------------
SHARD_CALLS = [  # (m, name, call(handle, pattern, flags), oracle)
    (14, "lp k=5", lambda h, p, f: h.search_levenshtein(p, 5, LP | f),
     lambda p, hay: oracle.levenshtein_lp_raw(p, hay, 5)),
    (36, "lp window 48", lambda h, p, f: h.search_levenshtein(p, 12, LP | f),
     lambda p, hay: oracle.levenshtein_lp_raw(p, hay, 12)),
    (38, "lp tile", lambda h, p, f: h.search_levenshtein(p, 12, LP | f),
     lambda p, hay: oracle.levenshtein_lp_raw(p, hay, 12)),
    (30, "generic-lp", lambda h, p, f: h.search_generic(p, 0, 20, 0, 20, LP | f),
     lambda p, hay: oracle.generic_lp_raw(p, hay, 0, 20, 0, 20)),
    (20, "generic-lp mixed", lambda h, p, f: h.search_generic(p, 2, 1, 1, 3, LP | f),
     lambda p, hay: oracle.generic_lp_raw(p, hay, 2, 1, 1, 3)),
    (66, "generic-ngrams", lambda h, p, f: h.search_generic(p, 20, 0, 0, 20, f),
     lambda p, hay: oracle.generic_ngrams_raw(p, hay, 20, 0, 0, 20)),
    (40, "generic-ngrams mixed", lambda h, p, f: h.search_generic(p, 2, 2, 2, 4, f),
     lambda p, hay: oracle.generic_ngrams_raw(p, hay, 2, 2, 2, 4)),
]


@pytest.mark.parametrize("nshards", [2, 3, 7])
def test_lp_generic_sharded_union_equals_whole(cuda_device, nshards):
    """The union of the shards' raw streams is the whole sequence's, for LP and generic searches, with near-matches
    across every seam at the deltas of test_sharded_union_equals_whole."""
    rng = np.random.default_rng(70 + nshards)
    n = (1 << 15) + 5
    alpha = np.frombuffer(ASCII, dtype=np.uint8)
    hay = alpha[rng.integers(0, len(alpha), size=n)].copy()
    pats = [bytes(alpha[rng.integers(0, len(alpha), size=m)]) for m, _, _, _ in SHARD_CALLS]
    for q, p in enumerate(pats):
        for _ in range(3):
            v = mutate(rng, p, ASCII, int(rng.integers(0, 4)))
            pos = int(rng.integers(100, n - 200))
            hay[pos:pos + len(v)] = np.frombuffer(v, dtype=np.uint8)
    bounds = [((n * i // nshards) // 16) * 16 for i in range(nshards)] + [n]
    for si, b in enumerate(bounds[1:-1]):
        for j, delta in enumerate((-1, 0, 1, -2, -4)):
            for q, p in enumerate(pats):
                pos = b + delta - len(p) // 2 * (q % 3 == 0) - len(p) * (q % 3 == 1) + 131 * (j - 2) * (q + 1)
                hay[pos:pos + len(p)] = np.frombuffer(p, dtype=np.uint8)
    halo = max(m for m, _, _, _ in SHARD_CALLS) + 20
    for (m, name, call, ref), p in zip(SHARD_CALLS, pats):
        whole = sorted(tup(ref(p, hay)))
        assert len(whole) >= 3 * nshards, name
        union = []
        for i in range(nshards):
            lo, hi = bounds[i], bounds[i + 1]
            blo = max(0, lo - halo) // 16 * 16
            hs = F.Haystack.from_host(hay[blo:min(n, hi + halo)], buf_lo=blo, global_len=n, own_lo=lo, own_hi=hi)
            res = call(hs, p, F.F_NO_FINAL)
            union += res.triples(F.RAW)
            res.close()
            hs.close()
        assert sorted(union) == whole, name


def test_lp_generic_at_64_bit_offsets(cuda_device):
    """An interior shard at global offsets up to 2^44 reports what the same bytes report at offset 0, shifted: LP
    searches with k >= 5 (streaming, window 48, tile kernel, through the survivor-list overflow) and generic searches
    with limits of 20, raw and final."""
    rng = np.random.default_rng(44)
    n = 20000
    alpha = np.frombuffer(ASCII, dtype=np.uint8)
    hay = alpha[rng.integers(0, len(alpha), size=n)].copy()
    pats = [bytes(alpha[rng.integers(0, len(alpha), size=m)]) for m, _, _, _ in SHARD_CALLS]
    for p in pats:
        for _ in range(4):
            v = mutate(rng, p, ASCII, int(rng.integers(0, 4)))
            pos = int(rng.integers(300, n - 400))
            hay[pos:pos + len(v)] = np.frombuffer(v, dtype=np.uint8)
    lo, hi = 256, n - 256
    a = F.Haystack.from_host(hay, buf_lo=0, global_len=n + (1 << 20), own_lo=lo, own_hi=hi)
    calls = [(p, lambda h, p, c=call: c(h, p, 0)) for (_, _, call, _), p in zip(SHARD_CALLS, pats)]
    calls.append((pats[0], lambda h, p: h.search_levenshtein(p, 5, LP | F.F_TINY_LIST)))
    want = []
    for p, call in calls:
        r = call(a, p)
        want.append((r.triples(F.RAW), r.triples(F.FINAL), launches(r)))
        assert len(want[-1][0]) >= 4
        r.close()
    for shift in SHIFTS:
        b = F.Haystack.from_host(hay, buf_lo=shift, global_len=shift + n + (1 << 20), own_lo=shift + lo,
                                 own_hi=shift + hi)
        for (p, call), (raw, fin, nl) in zip(calls, want):
            r = call(b, p)
            assert sorted(r.triples(F.RAW)) == sorted((s + shift, e + shift, d) for s, e, d in raw), hex(shift)
            assert r.triples(F.FINAL) == [(s + shift, e + shift, d) for s, e, d in fin], hex(shift)
            r.close()
        b.close()
    a.close()
