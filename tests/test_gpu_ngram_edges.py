"""The n-gram Levenshtein route (the benchmarked path) at its margins: the q-sample lemma of k_filter_sampled, every
byte offset of k_filter_dense / k_filter_dense2, the modes and slot size of k_verify_lev / k_verify_hits, and the
hand-over from k_post to the host and from the output buffer to a larger one.  Every search is compared with the
oracle twice: the raw stream element by element with its (n-gram, idx) anchors, and the final list.

Which path ran is read from stats() ("route", "n_launches": filter + verify + k_post per attempt) and from
Haystack.debug_counters(), the counters of the last attempt: word 0 counts raw records, word 3 marked granules, word
5 is 1 iff k_post consolidated the list (at most 16 384 records), word 7 counts list hits (k_verify_hits; 0 in
granule mode) and word 14 the keys k_post orders (one per warp for a match that several lanes found)."""
import numpy as np
import pytest

import oracle
from corpus import ASCII, DNA, make_corpus, mutate
from fuzzysearch_b200 import _native as F
from parity import tup

pytestmark = pytest.mark.gpu

SAMPLED, DENSE = "ngrams/sampled-filter", "ngrams/dense-filter"
ATTEMPT = 3            # launches per attempt: filter, verify, k_post
POST_MAX = 16384       # longest raw list k_post consolidates (post_kernels.cuh: kPostMax)
OUT_CAP = 1 << 16      # records the output buffer of a new handle holds
HIT_SLOT = 144         # k_verify_hits runs iff m + 2k + 8 fits this slot (kernels.cuh: kHitSlotBytes)
ROUND = 1024           # keys per round of k_post's sweep (kPostThreads)


# ---- helpers ---------------------------------------------------------------------------------------------------
def anchored(res):
    s, e, d, ng, ix = res.arrays(F.RAW, anchors=True)
    return list(zip(ng.tolist(), ix.tolist(), s.tolist(), e.tolist(), d.tolist()))


def oracle_anchored(pat, hay, k):
    raw, ng, ix = oracle.levenshtein_ngrams_raw(pat, hay, k, with_anchor=True)
    return [(int(a), int(b)) + t for a, b, t in zip(ng, ix, tup(raw))], raw


def check(res, pat, hay, k):
    """Raw stream with anchors element by element, and the final list, against the oracle -> the oracle's records."""
    want, raw = oracle_anchored(pat, hay, k)
    assert anchored(res) == want
    assert res.triples(F.FINAL) == tup(oracle.consolidate(raw))
    return want


def counters(hs):
    c = hs.debug_counters()
    return {"out": c[0], "gran": c[3], "post": c[5], "hits": c[7], "keys": c[14]}


def two_bit(hay):
    """The host's choice of k_filter_dense2 (api.cu: sample_collision_prob): collision probability >= 0.15 over the
    whole buffer, or over 16 blocks of 4 KiB of a longer one."""
    h = np.asarray(hay, dtype=np.uint8)
    if h.size > 16 * 4096:
        h = np.concatenate([h[((h.size - 4096) // 15 * i) & ~15:][:4096] for i in range(16)])
    p = np.bincount(h, minlength=256) / max(h.size, 1)
    return float((p * p).sum()) >= 0.15


def put(hay, pos, v):
    hay[pos:pos + len(v)] = np.frombuffer(bytes(v), dtype=np.uint8)


def random_text(rng, alphabet, n):
    alpha = np.frombuffer(alphabet, dtype=np.uint8)
    return alpha[rng.integers(0, len(alpha), size=n)].copy()


# ---- 1. k_filter_sampled at the lemma's margin ----------------------------------------------------------------
def aligned_hits(pat, hay, start, end):
    """(aligned words of H[start:end] equal to a 4-gram of P, aligned words in it)."""
    grams = {bytes(pat[o:o + 4]) for o in range(len(pat) - 3)}
    words = range((start + 3) // 4 * 4, end - 3, 4)
    return sum(bytes(hay[w:w + 4]) in grams for w in words), len(words)


def one_word_plant(rng, pat, k, r):
    """P with k deletions, each inside a different aligned word of an occurrence starting at r (mod 4): all of its
    aligned words are broken but one, or two where the alignment fits k + 2 words -> (occurrence, the offsets in it
    of the n-grams that stay intact)."""
    m, L = len(pat), len(pat) // (k + 1)
    words = list(range((-r) % 4, m - k - 3, 4))
    broken = sorted(rng.choice(len(words), size=k, replace=False))
    gaps = [words[w] + int(rng.integers(1, 4)) for w in broken]        # the deleted byte sat before occ[gap]
    dels = {g + i for i, g in enumerate(gaps)}                          # as indices of P
    occ = bytes(c for i, c in enumerate(pat) if i not in dels)
    intact = [j * L - sum(d < j * L for d in dels) for j in range(m // L)
              if not any(j * L <= d < j * L + L for d in dels)]
    return occ, intact


def sampled_margin_input(alphabet, m, k, seed):
    """Occurrences of one_word_plant at every start mod 4, with an intact n-gram anchored at granule offsets 0, 1,
    62 and 63.  The start's alignment and the anchor's offset are tied through the n-gram offsets, so each pair
    (start mod 4, anchor offset) that some layout reaches gets an occurrence, and every start residue and every
    anchor offset must be reached."""
    rng = np.random.default_rng(seed)
    for _ in range(100):   # (a pattern with runs, e.g. TTTT on DNA, keeps a word intact whatever is deleted)
        pat = bytes(random_text(rng, alphabet, m))
        hay = random_text(rng, alphabet, 128 * 16 + 256)
        placed = set()
        for slot, (r, t) in enumerate((r, t) for r in range(4) for t in (0, 1, 62, 63)):
            base = 128 + 128 * slot
            for _ in range(100):
                occ, intact = one_word_plant(rng, pat, k, r)
                a = next((a for a in intact if (t - a - r) % 4 == 0), None)
                if a is None:
                    continue
                s0 = base + (t - a) % 64
                put(hay, s0, occ)
                hits, words = aligned_hits(pat, hay, s0, s0 + len(occ))
                if hits == words - k:   # no broken word equals another 4-gram of P by chance
                    placed.add((r, t))
                    break
        if {r for r, _ in placed} == {0, 1, 2, 3} and {t for _, t in placed} == {0, 1, 62, 63}:
            return pat, hay
    raise AssertionError("no pattern reaches every start residue and anchor offset")


TIGHT = [(m, k) for k, lo in ((1, 12), (2, 17), (3, 22), (4, 27)) for m in range(lo, lo + 4)]
BELOW = [(11, 1), (16, 2), (21, 3), (26, 4)]


@pytest.mark.parametrize("alphabet", [ASCII, DNA])
@pytest.mark.parametrize("m,k", TIGHT + BELOW)
def test_sampled_filter_at_the_lemma_margin(cuda_device, alphabet, m, k):
    """k_filter_sampled runs iff floor((m-k-3)/4) >= k+1: an occurrence of m - k bytes then holds k + 1 aligned
    words (at some alignments k + 2), and k deletions can break all but one.  Such occurrences sit at every start
    mod 4 with their anchor at granule offsets 0, 1, 62 and 63; the one intact word must mark the anchor's granule.
    One step below the margin the host must take the dense filter even when the sampled one is forced."""
    pat, hay = sampled_margin_input(alphabet, m, k, 1000 * k + m + len(alphabet))
    hs = F.Haystack.from_host(hay)
    res = hs.search_levenshtein(pat, k, F.F_FORCE_SAMPLED)
    want = check(res, pat, hay, k)
    tight = (m, k) in TIGHT
    assert res.stats()["route"] == (SAMPLED if tight else DENSE)
    assert res.stats()["n_launches"] == ATTEMPT
    if tight:
        single = {}   # start mod 4 -> anchor offsets of the records whose occurrence holds k + 1 words, one intact
        for _, idx, s, e, _ in want:
            hits, words = aligned_hits(pat, hay, s, e)
            if words == k + 1 and hits == 1:
                single.setdefault(s % 4, set()).add(idx % 64)
        fits = {r for r in range(4) if len(range((-r) % 4, m - k - 3, 4)) == k + 1}
        assert fits and set(single) >= fits, (single, fits)      # otherwise the plants have gone slack
    res.close()
    hs.close()


# ---- 2. k_filter_dense / k_filter_dense2 at every byte offset -------------------------------------------------------
DNA_EXTRA = b"ACGTACGTACGTACGTACGTACGTACGTNacgt"   # mostly ACGT; N and lowercase alias A, C, G, T in the 2-bit codes


def dense_input(alphabet, L, n, seed):
    """k = 1, m = 2L.  Exact copies of P whose first n-gram is anchored at every offset 0..15 of a vector, at the
    last bytes before a warp's 512 B (lane 31 reads ahead), before each 16 KiB tile, and at the buffer's end."""
    rng = np.random.default_rng(seed)
    m = 2 * L
    pat = bytearray(random_text(rng, alphabet if alphabet != DNA_EXTRA else DNA, m))
    if alphabet == DNA_EXTRA:
        pat[1], pat[-2] = ord("N"), ord("c")
    pat = bytes(pat)
    hay = random_text(rng, alphabet, n)
    starts = [1024 + 33 * i for i in range(16)]                       # offsets 0..15 of a vector
    starts += [512 * w - (w - 3) for w in range(4, 12)]               # 1..8 bytes before a warp's block
    starts += [(1 << 14) - 3, (2 << 14) - 7]                          # before each 16 KiB tile
    starts += [n - m - 40, n - m]                                     # the buffer's last vectors, a copy ending at N
    for s in starts:
        put(hay, s, pat)
    put(hay, n - m - 20, pat[:-1] + bytes([pat[0]]))                  # an edit on the last character
    return pat, hay


@pytest.mark.parametrize("alphabet,L", [(ASCII, L) for L in (3, 4, 5, 7, 8, 10)] +
                         [(DNA_EXTRA, L) for L in range(3, 9)])
def test_dense_filters_at_every_byte_offset(cuda_device, alphabet, L):
    """k_filter_dense in its four modes (q = 3; 4; 5, 7; 8 and L = 10 > 8) on text, k_filter_dense2 (q = 3..8) on
    DNA with N and lowercase bytes in the text and the pattern (the 2-bit aliasing may only add candidates), at buffer
    lengths 1, 13 and 15 (mod 16), through the hit list and through granule mode (FZB_F_TINY_LIST: the hit list
    holds 8 entries, overflows, and the search is repeated in granule mode)."""
    k = 1
    for r in (1, 13, 15):
        n = 33776 + r
        pat, hay = dense_input(alphabet, L, n, 100 * L + r)
        assert two_bit(hay) == (alphabet != ASCII)
        hs = F.Haystack.from_host(hay)
        for extra in (0, F.F_TINY_LIST):
            res = hs.search_levenshtein(pat, k, F.F_FORCE_DENSE | extra)
            want = check(res, pat, hay, k)
            assert len(want) >= 30
            c = counters(hs)
            assert res.stats()["route"] == DENSE
            if extra:
                # (the granule list holds 8 too: a third attempt sweeps the bitmap the second one left set)
                assert res.stats()["n_launches"] in (2 * ATTEMPT, 3 * ATTEMPT) and c["hits"] == 0
            else:
                assert res.stats()["n_launches"] == ATTEMPT and c["hits"] >= len(want) // 2 and c["gran"] == 0
            res.close()
        hs.close()


# ---- 3. k_verify_lev / k_verify_hits at their limits ---------------------------------------------------------------
def verify_input(alphabet, m, k, n, seed):
    """make_corpus's plants (up to k + 1 edits, clusters, both global ends) plus copies with an edit on the last
    character (substituted, deleted, preceded by an insertion) and with k edits, one of them on the last character."""
    pat, hay, _ = make_corpus(seed, n, alphabet, m, 6, k + 1)
    rng = np.random.default_rng(seed)
    other = bytes([c for c in alphabet if c != pat[-1]][:1])
    plants = [pat[:-1] + other, pat[:-1], pat[:-1] + other + pat[-1:],
              mutate(rng, pat[:-1], alphabet, k - 1) + other]
    step = (n - 4 * m) // (len(plants) + 1)
    for i, v in enumerate(plants):
        put(hay, 2 * m + step * i + int(rng.integers(0, 64)), v)
    return pat, hay


VERIFY = [  # (alphabet, m, k): the verify mode, the expansion routine, the short / long variant, the hit slot
    (ASCII, 48, 2),    # m - L = 32: mode 0, the right sub-pattern fills the 32-bit word
    (ASCII, 49, 2),    # m - L = 33: mode 1 (64-bit words)
    (ASCII, 64, 1),    # mode 0 at m = 64
    (ASCII, 64, 2),    # mode 1 at m = 64
    (ASCII, 65, 2),    # mode 2 (cell by cell)
    (ASCII, 80, 4),    # mode 2, sub-patterns of 16: expand_uni_reg
    (ASCII, 68, 3),    # mode 2, sub-patterns of 17: expand_dp
    (ASCII, 18, 1),    # sub-patterns of 9, 10, 11 around max(2k, 10) = 10: short, short, long
    (ASCII, 20, 1),
    (ASCII, 22, 1),
    (ASCII, 77, 6),    # 11, 12, 13 around max(2k, 10) = 12 (expand_uni_reg)
    (ASCII, 84, 6),
    (ASCII, 91, 6),
    (ASCII, 170, 9),   # 17, 18, 19 around 18 (expand_dp short / long)
    (ASCII, 180, 9),
    (ASCII, 190, 9),
    (DNA, 120, 8),     # m + 2k + 8 = 144: the hit slot exactly
    (DNA, 128, 4),     # 144
    (DNA, 129, 4),     # 145: granule mode
    (ASCII, 255, 84),  # the largest halo (m + k = 339) at the first and last granule of the buffer
]


@pytest.mark.parametrize("alphabet,m,k", VERIFY)
def test_verify_kernels_at_their_limits(cuda_device, alphabet, m, k):
    """Every verify mode and expansion routine at its boundary, with edits on the pattern's last character (the top
    bit of the word), on the route the host picks and on the dense route (k_verify_hits iff m + 2k + 8 <= 144),
    then on an interior shard with the smallest halo (the lane and granule windows end at the buffer's edges)."""
    n = 8192
    pat, hay = verify_input(alphabet, m, k, n, 7 * m + k)
    hs = F.Haystack.from_host(hay)
    for flags in (0, F.F_FORCE_DENSE):
        res = hs.search_levenshtein(pat, k, flags)
        want = check(res, pat, hay, k)
        assert len(want) >= 6
        c = counters(hs)
        if res.stats()["route"] == DENSE and m + 2 * k + 8 <= HIT_SLOT:
            assert c["hits"] > 0 and c["gran"] == 0
        else:
            assert c["hits"] == 0 and c["gran"] > 0
        assert res.stats()["n_launches"] == ATTEMPT
        res.close()
    hs.close()
    L = m // (k + 1)
    last = (m // L - 1) * L   # offset of the last n-gram in P
    lo, hi = n // 3 + 1, 2 * n // 3 + 15
    geometries = [(lo, hi), (lo + 4 * m, hi - 4 * m)]
    for p0 in (lo - 1, hi - 1, lo + 4 * m - last, hi - 4 * m - last):  # anchors lo - 1, hi - 1 (first n-gram) and,
        put(hay, p0, pat)                                              # in the inner geometry, lo and hi (last one)
    want, _ = oracle_anchored(pat, hay, k)
    halo = m + k
    for glo, ghi in geometries:
        blo = (glo - halo) // 16 * 16
        sh = F.Haystack.from_host(hay[blo:ghi + halo], buf_lo=blo, global_len=n, own_lo=glo, own_hi=ghi)
        mine = sorted(w for w in want if glo <= w[1] < ghi)
        assert {glo - 1, ghi - 1, glo, ghi} & {w[1] for w in want}
        for flags in (0, F.F_FORCE_DENSE):
            res = sh.search_levenshtein(pat, k, flags | F.F_NO_FINAL)
            assert sorted(anchored(res)) == mine
            res.close()
        sh.close()


def test_same_match_through_several_ngrams(cuda_device):
    """Exact copies found through every n-gram: within one warp pass (m = 20, k = 2: anchors 6 bytes apart), the
    lanes share one key, so k_post orders fewer keys than there are records; through n-grams in different granules
    (m = 200, k = 1: anchors 100 bytes apart) every record has its key.  The final list is the oracle's either way."""
    rng = np.random.default_rng(3)
    for m, k in ((20, 2), (200, 1)):
        pat = bytes(random_text(rng, ASCII, m))
        hay = random_text(rng, ASCII, 1 << 14)
        for i in range(20):
            put(hay, 256 + 640 * i + (i % 2) * 13, pat)
        hs = F.Haystack.from_host(hay)
        res = hs.search_levenshtein(pat, k, F.F_FORCE_SAMPLED)
        want = check(res, pat, hay, k)
        c = counters(hs)
        assert res.stats()["route"] == SAMPLED and c["post"] == 1 and c["out"] == len(want) >= 20 * (k + 1)
        if m == 20:
            assert c["keys"] < c["out"]
        res.close()
        hs.close()


# ---- 4. hand-over: k_post -> host, output buffer -> a larger one ----------------------------------------------------
def copies_input(pat, copies, half, seed, gap=4):
    """`copies` exact copies of P, `gap` random bytes apart, then `half` copies with the last character substituted
    (found through the first n-gram only when k = 1)."""
    rng = np.random.default_rng(seed + 1)   # (not the pattern's stream)
    m = len(pat)
    hay = random_text(rng, ASCII, (copies + half) * (m + gap) + 64)
    other = bytes([c for c in ASCII if c != pat[-1]][:1])
    for i in range(copies + half):
        put(hay, 32 + i * (m + gap), pat if i < copies else pat[:-1] + other)
    return hay


@pytest.mark.parametrize("records", [POST_MAX, POST_MAX + 1])
@pytest.mark.parametrize("route", ["levenshtein", "exact", "hamming"])
def test_post_hand_over(cuda_device, route, records):
    """k_post takes lists of up to 16 384 raw records; one more goes to the host twin (consolidate_recs), which must
    give the same final list: on the consolidating route and on the unconsolidated ones (exact, Hamming)."""
    rng = np.random.default_rng(records)
    if route == "levenshtein":   # 2 records per exact copy, 1 per copy with its last character substituted
        pat = bytes(random_text(rng, ASCII, 12))
        hay = copies_input(pat, records // 2, records % 2, records)
    else:
        pat = bytes(random_text(rng, ASCII, 16))
        hay = copies_input(pat, records, 0, records)
    hs = F.Haystack.from_host(hay)
    if route == "levenshtein":
        res = hs.search_levenshtein(pat, 1)
        want = check(res, pat, hay, 1)
        assert len(want) == records
    else:
        res = hs.search_exact(pat) if route == "exact" else hs.search_hamming(pat, 2)
        cpu = [(s, s + len(pat), 0) for s in oracle.search_exact(pat, hay)] if route == "exact" \
            else tup(oracle.substitutions(pat, hay, 2))
        assert len(cpu) == records
        assert sorted(res.triples(F.RAW)) == cpu and res.triples(F.FINAL) == cpu
    c = counters(hs)
    assert c["out"] == records and c["post"] == (records <= POST_MAX)
    assert res.stats()["n_launches"] == ATTEMPT
    res.close()
    hs.close()


def periodic_input(regions, seed):
    """Random text with periodic regions (period 5) of the given lengths, and a pattern of the same period: every
    region is one group of overlapping matches whose best records tie on (dist, length)."""
    rng = np.random.default_rng(seed)
    unit = bytes(random_text(rng, ASCII, 5))
    pat = (unit * 4)[:20]
    hay = random_text(rng, ASCII, sum(regions) + 200 * len(regions) + 200)
    pos = 200
    for r in regions:
        put(hay, pos, (unit * (r // 5 + 1))[:r])
        pos += r + 200
    return pat, hay


@pytest.mark.parametrize("regions", [[20000], [6000, 700, 6500, 300, 1300]])
def test_post_groups_across_rounds(cuda_device, regions):
    """k_post sweeps the sorted keys 1 024 per round, carrying the hull and the group count between rounds: one group
    spanning every round, and groups straddling the round boundaries (more than 1 024 distinct records each).  Within
    a group the best records tie on (dist, length); the winner is the smallest (start, end)."""
    pat, hay = periodic_input(regions, len(regions))
    hs = F.Haystack.from_host(hay)
    res = hs.search_levenshtein(pat, 2)
    want = check(res, pat, hay, 2)
    fin, groups = oracle.consolidate(np.array([w[2:] for w in want]), with_groups=True)
    assert len(fin) == len(regions)
    distinct = [len({w[2:] for w, g in zip(want, groups) if g == i}) for i in range(len(regions))]
    assert max(distinct) > 2 * ROUND if len(regions) == 1 else sum(d > ROUND for d in distinct) >= 2, distinct
    c = counters(hs)
    assert c["post"] == 1 and c["out"] == len(want) <= POST_MAX
    res.close()
    hs.close()


@pytest.mark.parametrize("records", [OUT_CAP, OUT_CAP + 1])
def test_output_buffer_growth(cuda_device, records):
    """A raw stream longer than the output buffer (65 536 records on a new handle) grows it and repeats the attempt;
    a second search on the same handle runs once.  Both go to the host's consolidation."""
    pat = bytes(random_text(np.random.default_rng(5), ASCII, 12))
    hay = copies_input(pat, records // 2, records % 2, 5)
    hs = F.Haystack.from_host(hay)
    first = hs.search_levenshtein(pat, 1)
    want = check(first, pat, hay, 1)
    assert len(want) == records and counters(hs)["post"] == 0
    again = hs.search_levenshtein(pat, 1)
    check(again, pat, hay, 1)
    assert again.stats()["n_launches"] == ATTEMPT
    assert first.stats()["n_launches"] == (ATTEMPT if records <= OUT_CAP else 2 * ATTEMPT)
    first.close()
    again.close()
    hs.close()


# ---- 5. shards --------------------------------------------------------------------------------------------------
SHARD_PATHS = [  # (name, alphabet, m, k, flags)
    ("sampled", ASCII, 20, 2, F.F_FORCE_SAMPLED),
    ("dense, granules", ASCII, 100, 20, F.F_FORCE_DENSE),
    ("dense, hit list", ASCII, 20, 2, F.F_FORCE_DENSE),
    ("dense2, hit list", DNA, 20, 2, F.F_FORCE_DENSE),
]


@pytest.mark.parametrize("nshards", [2, 3, 7])
def test_ngram_sharded_union_equals_whole(cuda_device, nshards):
    """The union of the shards' raw streams (with anchors) is the whole sequence's, on the sampled, dense, dense2
    and hit-list paths.  The seams sit at offsets 1 and 15 (mod 16) and 63 (mod 64); copies are anchored at the last
    position of one shard and at the first of the next (one haystack each), through the first and the last n-gram."""
    n = (1 << 14) + 5
    bounds = [0] + [(n * i // nshards) // 64 * 64 + (1, 15, 63)[i % 3] for i in range(1, nshards)] + [n]
    for name, alphabet, m, k, flags in SHARD_PATHS:
        L = m // (k + 1)
        for side in (0, 1):
            rng = np.random.default_rng(nshards * 10 + side)
            pat = bytes(random_text(rng, alphabet, m))
            hay = random_text(rng, alphabet, n)
            for si, b in enumerate(bounds[1:-1]):
                j = (si + side) % (m // L)
                v = bytearray(pat)
                if si % 2:   # a substitution outside the anchored n-gram
                    v[(j * L + L) % m] = next(c for c in alphabet if c != pat[(j * L + L) % m])
                put(hay, b - 1 + side - j * L, v)
            whole, _ = oracle_anchored(pat, hay, k)
            assert {b - 1 + side for b in bounds[1:-1]} <= {w[1] for w in whole}, name
            union = []
            for i in range(nshards):
                lo, hi = bounds[i], bounds[i + 1]
                blo = max(0, lo - (m + k)) // 16 * 16
                hs = F.Haystack.from_host(hay[blo:min(n, hi + m + k)], buf_lo=blo, global_len=n, own_lo=lo,
                                          own_hi=hi)
                res = hs.search_levenshtein(pat, k, flags | F.F_NO_FINAL)
                union += anchored(res)
                res.close()
                hs.close()
            assert sorted(union) == sorted(whole), name
