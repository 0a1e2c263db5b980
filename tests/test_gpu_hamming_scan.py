"""k_hamming_count, the scan of the substitutions-only search, at the geometry of its tiles, its ring and its counters:
256-row tiles of 128-byte rows loaded by TMA behind an 8-row halo atom, a 2-stage mbarrier ring on a persistent grid,
7 warm-up words from the previous row, two or three bit slices of counters over a 256-bucket hashed match table, and
out-of-bounds rows that read as zeros.

What the scan decides is the set of marked granules, and stats()["n_candidates"] counts them.  The tests restate
that set in numpy from the definition of the filter (hamming_marks below: per alignment class and first counted word,
the running number of counted words whose hash bucket equals that of the pattern 4-gram at their offset, firing
where bias + count carries out of its slices; a row holding a fire marks the starts whose counted words can reach
it) and compare the count.  The raw list is compared with the oracle element for element and with the brute-force
kernel (k_hamming_scan).  `small` replays every body on the emulated device, whose grid is 4 CTAs."""
import numpy as np
import pytest

import oracle
from corpus import ASCII, DNA
from fuzzysearch_b200 import _native as F
from parity import tup

pytestmark = pytest.mark.gpu

HAMMING = "hamming"
ROW = 128                   # bytes per row = per thread (ham_kernels.cuh: kHcRowBytes)
TILE_ROWS = 256             # rows per tile after the 8-row halo atom (kHcThreads)
TILE = TILE_ROWS * ROW      # 32 KiB of buffer per tile
GRID_PASS = 2 * 132         # tiles of one pass of the grid on an H100: two CTAs per SM
EMU_PASS = 4                # the emulated device: 2 SMs, 2 CTAs per SM
HASH = 0x9E3779B1           # ham_recur.h: kHcHashMul
HASH_INV = pow(HASH, -1, 1 << 32)


def bucket(w):
    """hc_bucket of u32 words (an int or an array): the top byte of w * HASH mod 2^32."""
    return ((np.asarray(w, dtype=np.uint64) * HASH) & 0xFFFFFFFF) >> 24


def gram(pat, o):
    return int.from_bytes(bytes(pat[o:o + 4]), "little")


def layout(m, k, slices=None):
    """-> (Wc, threshold T, slices S, bias) of the counting filter; `slices` overrides fzb_search_hamming's choice."""
    Wc = min((m - 3) // 4, 8)
    T = Wc - k
    S = slices or (2 if T <= 4 else 3)
    bias = (1 << S) - T
    assert T >= 1 and 0 <= bias < (1 << S), (m, k, S)
    return Wc, T, S, bias


def scanned_words(buf):
    """The little-endian u32 words of every row the scan reads: ceil(ceil(len/128) / 256) whole tiles, zeros past
    the buffer's end (its zero padding and the out-of-bounds rows of the last tile)."""
    n = len(buf)
    nrows = (n + ROW - 1) // ROW
    ntiles = (nrows + TILE_ROWS - 1) // TILE_ROWS
    b = np.zeros(ntiles * TILE, dtype=np.uint8)
    b[:n] = np.frombuffer(bytes(buf), dtype=np.uint8)
    return b.view("<u4")


def fire_words(pat, k, buf, slices=None):
    """Boolean per scanned word: some occurrence's counters carry out there.  For an occurrence with first counted
    word t0 and class o0, c_j counts the i <= j with bucket(word t0+i) == bucket(P[o0+4i : o0+4i+4]); it fires at word
    t0+j where that holds and floor((bias + c_j) / 2^S) goes up.  Words before the buffer are zeros."""
    m = len(pat)
    Wc, _, S, bias = layout(m, k, slices)
    bw = bucket(scanned_words(buf)).astype(np.int16)
    nw = bw.size
    z = int(bucket(0))
    ext = np.concatenate([np.full(7, z, np.int16), bw, np.full(8, z, np.int16)])  # ext[u]: word u - 7
    n0 = nw + 7                                   # first counted words t0 = -7 .. nw - 1, at u = t0 + 7
    fire = np.zeros(ext.size, dtype=bool)         # fire[u]: word u - 7
    top = (1 << S) - 1
    for o0 in range(4):                           # class by class: memory stays a few arrays of the text's size
        c = np.full(n0, bias, dtype=np.int16)     # bias + c_j of every occurrence of the class
        for j in range(Wc):
            hit = ext[j:j + n0] == int(bucket(gram(pat, o0 + 4 * j)))
            c += hit
            fire[j:j + n0] |= hit & ((c & top) == 0)
    return fire[7:7 + nw]


def flagged_rows(pat, k, buf, slices=None):
    return np.nonzero(fire_words(pat, k, buf, slices).reshape(-1, 32).any(axis=1))[0].astype(np.int64)


def mark_ranges(pat, k, buf, buf_lo, own_lo, own_hi, slices=None):
    """The inclusive global ranges of starts the flagged rows mark, clipped to [own_lo, own_hi) as mark_range_inline
    clips them (empty ones dropped)."""
    Wc = layout(len(pat), k, slices)[0]
    r = flagged_rows(pat, k, buf, slices)
    lo = np.maximum(np.maximum(4 * (32 * r - Wc + 1) - 3, 0) + buf_lo, own_lo)
    hi = np.minimum(4 * (32 * r + 31) + buf_lo, own_hi - 1)
    keep = lo <= hi
    return lo[keep], hi[keep]


def hamming_marks(pat, k, buf, buf_lo, own_lo, own_hi, slices=None):
    """The granules k_hamming_count marks on the buffer `buf` that starts at global position buf_lo."""
    lo, hi = mark_ranges(pat, k, buf, buf_lo, own_lo, own_hi, slices)
    g0, g1 = (lo - buf_lo) >> 6, (hi - buf_lo) >> 6
    parts = [(g0 + d)[g0 + d <= g1] for d in range(int((g1 - g0).max()) + 1 if g0.size else 0)]
    return set(np.unique(np.concatenate(parts)).tolist()) if parts else set()


def random_text(rng, n, alphabet=ASCII):
    alpha = np.frombuffer(alphabet, dtype=np.uint8)
    return alpha[rng.integers(0, len(alpha), size=n)].copy()


def subs(rng, pat, nsub):
    """P with exactly `nsub` substitutions."""
    v = bytearray(pat)
    for i in rng.choice(len(v), size=min(nsub, len(v)), replace=False):
        v[i] = (v[i] + int(rng.integers(1, 256))) % 256
    return bytes(v)


def put(hay, pos, v):
    if pos < 0:
        return
    v = np.frombuffer(bytes(v), dtype=np.uint8)[:max(0, len(hay) - pos)]
    hay[pos:pos + len(v)] = v


def seam_plants(rng, hay, pat, k, seams, lo=0):
    """At every seam b (buffer offsets; the buffer starts at hay[lo]) one occurrence of each alignment class, in a
    random order over four slots: ending in the row before the seam, straddling it (its counted words on both sides,
    so the row after the seam warms up on the row before it), and two starting in the row after it.  Each has 0 to
    k + 1 substitutions."""
    m = len(pat)
    Wc = min((m - 3) // 4, 8)
    for b in seams:
        a = rng.permutation(4)
        d = int(rng.integers(1, Wc + 1))
        for s in (b - 2 * m - 8 - a[0], b - 4 * d - a[1], b + m + a[2], b + 2 * m + 8 + a[3]):
            put(hay, lo + s, subs(rng, pat, int(rng.integers(0, k + 2))))


def end_plants(rng, hay, pat, k):
    """A copy at position 0; one with k + 1 substitutions and one with k near the end where they fit between the two
    ends; last, at the end, a copy ending at N if N is even, a prefix cut off by the end if N is odd (one buffer cannot
    end in both).  -> (a match starts at 0, a match ends at N): what the oracle list must hold."""
    n, m = len(hay), len(pat)
    put(hay, 0, pat)
    if n >= 4 * m + 16:
        put(hay, n - 3 * m - 9, subs(rng, pat, k + 1))
        put(hay, n - 2 * m - 5, subs(rng, pat, k))
    if n % 2 == 0:
        put(hay, n - m, pat)
    else:
        put(hay, n - m // 2, pat)
    return n >= 2 * m, n % 2 == 0 and n >= m


def check_ends(raw, n, ends):
    """The matches end_plants guarantees are in the list `raw` (ascending by start)."""
    at0, atn = ends
    assert not at0 or raw[0][0] == 0, n
    assert not atn or any(e == n for _, e, _ in raw), n


def tile_seams(n):
    return range(TILE, n, TILE)


def search_and_check(hs, pat, hay, k, flags=0, marks=None, ends=(False, False)):
    """One whole-sequence search: RAW against the oracle (holding the matches at the ends that `ends` promises),
    FINAL == RAW, the group rows' hulls the matches themselves, the candidate count against the restated marks, RAW
    against the brute-force kernel -> (marks, raw records)."""
    res = hs.search_hamming(pat, k, flags)
    st = res.stats()
    assert st["route"] == HAMMING
    raw = res.triples(F.RAW)
    assert raw == tup(oracle.substitutions(pat, hay, k)), len(hay)
    check_ends(raw, len(hay), ends)
    assert res.triples(F.FINAL) == raw, len(hay)
    assert res.group_rows().tolist() == [[s, e, d, s, e] for s, e, d in raw], len(hay)
    if marks is None:
        marks = hamming_marks(pat, k, hay, 0, 0, len(hay))
    assert st["n_candidates"] == len(marks), (len(hay), len(pat), k)
    res.close()
    dense = hs.search_hamming(pat, k, F.F_FORCE_DENSE)
    assert dense.triples(F.RAW) == raw, len(hay)
    dense.close()
    return len(marks), len(raw)


def test_buffer_lengths_around_tiles_and_grid_passes(cuda_device, small=False):
    """Buffers of every length mod 16 around one row, one and two tiles, and a handful around one, two (plus one) and
    three passes of the grid: a CTA refills stage 0 and waits on its second parity.  Occurrences of every class at
    every tile seam, at both ends, and a prefix cut off by the end."""
    rng = np.random.default_rng(21)
    m, k = 32, 3
    pat = bytes(random_text(rng, m, DNA))
    G = EMU_PASS if small else GRID_PASS
    big = [G * TILE, (2 * G + 1) * TILE, 3 * G * TILE]
    base = random_text(rng, big[-1] + 256, DNA)
    seam_plants(rng, base, pat, k, tile_seams(len(base)))
    for s in range(1000, len(base) - 1000, 9973):
        put(base, s, subs(rng, pat, int(rng.integers(0, k + 2))))
    lengths = [b + d for b in (ROW, TILE, 2 * TILE) for d in range(-8, 8)]
    lengths += [b + d for b in big for d in (-128, -1, 0, 1, 128)]
    marks = raw = 0
    for n in lengths:
        hay = base[:n].copy()
        ends = end_plants(rng, hay, pat, k)
        hs = F.Haystack.from_host(hay)
        got = search_and_check(hs, pat, hay, k, ends=ends)
        marks, raw = marks + got[0], raw + got[1]
        hs.close()
    assert marks > 0 and raw >= 2 * len(lengths)


# (m, k): Wc 1 (k = 0, m 7 to 10) to 8, thresholds T = Wc - k from 1 to 8, the slice boundary T = 4 (two slices)
# against T = 5 (three), double carries of two slices (k >= 4: m = 35 with k = 4..7, m = 23 with k = 4), m = 255
LAYOUTS = [(7, 0), (8, 0), (9, 0), (10, 0), (11, 1), (15, 0), (19, 2), (23, 4), (27, 1), (31, 3), (32, 3), (32, 2),
           (35, 7), (35, 6), (35, 5), (35, 4), (35, 3), (35, 2), (35, 1), (35, 0), (40, 0), (255, 7), (255, 2),
           (255, 0)]


def quiet_text(rng, n, pat, k):
    """Random ASCII none of whose aligned words falls in the bucket of a counted gram: only planted occurrences fire,
    even at threshold 1."""
    Wc = layout(len(pat), k)[0]
    hot = [int(bucket(gram(pat, o0 + 4 * i))) for o0 in range(4) for i in range(Wc)]
    hay = random_text(rng, n + 3)
    words = hay[:(n + 3) // 4 * 4].view("<u4")
    while True:
        bad = np.isin(bucket(words), hot)
        if not bad.any():
            return hay[:n].copy()
        words[bad] = random_text(rng, 4 * int(bad.sum())).view("<u4")


def double_carry(m, k):
    """Two slices carry twice in one field: threshold T <= 4 and T + 4 <= Wc counted words (k >= 4)."""
    Wc, T, S, _ = layout(m, k)
    return S == 2 and T + 4 <= Wc


def distinct_grams_pattern(rng, m, k):
    """A random ASCII pattern whose 4 * Wc counted grams fall in 4 * Wc different buckets, none of them the zero
    word's: a word equal to one of them adds to no other field, and the zeros past the end add to none."""
    Wc = layout(m, k)[0]
    while True:
        pat = bytes(random_text(rng, m))
        b = {int(bucket(gram(pat, o0 + 4 * i))) for o0 in range(4) for i in range(Wc)}
        if len(b) == 4 * Wc and int(bucket(0)) not in b:
            return pat


def carry_plants(hay, pat, k, rows):
    """The counted words of class 0 only (P[:4 Wc], word-aligned), placed so that the first carry lies in the last
    word of a row: the second carry of two slices, four counted words later, lies in the next row; three slices have
    none.  On quiet_text with a distinct_grams_pattern nothing else fires there, at any threshold."""
    Wc, T = layout(len(pat), k)[:2]
    for r in rows:
        put(hay, 4 * (32 * r + 32 - T), pat[:4 * Wc])


def test_counter_layouts(cuda_device, small=False):
    """Every (Wc, threshold, slices) layout the host picks, on text with planted variants and on two-letter text that
    repeats the pattern's grams.  Where two slices carry twice, copies placed so that the second carry flags a row of
    its own make the two layouts' counts differ, so the count also pins the slice choice of fzb_search_hamming."""
    rng = np.random.default_rng(22)
    n = TILE + 4321 if small else 3 * TILE + 4321
    differ = []
    for m, k in LAYOUTS:
        pat = distinct_grams_pattern(rng, m, k) if double_carry(m, k) else bytes(random_text(rng, m))
        hay = quiet_text(rng, n, pat, k)
        if double_carry(m, k):
            carry_plants(hay, pat, k, range(5, (n - 2 * ROW) // ROW, 23))
        for s in range(100, n - m - 100, 1531):
            put(hay, s, subs(rng, pat, int(rng.integers(0, k + 2))))
        seam_plants(rng, hay, pat, k, tile_seams(n))
        ends = end_plants(rng, hay, pat, k)
        hs = F.Haystack.from_host(hay)
        marks, raw = search_and_check(hs, pat, hay, k, ends=ends)
        assert marks > 0 and raw > 0, (m, k)
        if layout(m, k)[2] == 2 and marks != len(hamming_marks(pat, k, hay, 0, 0, n, slices=3)):
            differ.append((m, k))
        hs.close()
        ab_pat = bytes(random_text(rng, m, b"ab"))
        ab = random_text(rng, n // 3, b"ab")
        hs = F.Haystack.from_host(ab)
        search_and_check(hs, ab_pat, ab, k)
        hs.close()
    # every double-carry layout, (23, 4), (35, 4..7) and (255, 7), and only those
    assert differ == [(m, k) for m, k in LAYOUTS if double_carry(m, k)] and len(differ) == 6


@pytest.mark.parametrize("k", range(8))
def test_dispatch_boundary(cuda_device, k, small=False):
    """m = 4k + 7 counts (one launch more than the brute-force kernel), m = 4k + 6 is brute force, which reports no
    candidates; k = 7 counts and k = 8 does not.  Every side equals the oracle."""
    rng = np.random.default_rng(23 + k)
    n = TILE + 999 if small else 2 * TILE + 999
    hay = random_text(rng, n, DNA)
    for m, kk, counting in ((4 * k + 7, k, True), (4 * k + 6, k, False)) + \
            (((48, 7, True), (48, 8, False)) if k == 7 else ()):
        pat = bytes(random_text(rng, m, DNA))
        h = hay.copy()
        for s in range(50, n - m - 50, 777):
            put(h, s, subs(rng, pat, int(rng.integers(0, kk + 2))))
        ends = end_plants(rng, h, pat, kk)
        hs = F.Haystack.from_host(h)
        res = hs.search_hamming(pat, kk)
        dense = hs.search_hamming(pat, kk, F.F_FORCE_DENSE)
        st, sd = res.stats(), dense.stats()
        want = tup(oracle.substitutions(pat, h, kk))
        assert res.triples(F.RAW) == want == dense.triples(F.RAW), (m, kk)
        check_ends(want, n, ends)
        assert st["route"] == sd["route"] == HAMMING
        assert sd["n_candidates"] == 0
        if counting:
            assert st["n_launches"] == sd["n_launches"] + 1, (m, kk)
            assert st["n_candidates"] == len(hamming_marks(pat, kk, h, 0, 0, n)) > 0, (m, kk)
        else:
            assert st["n_launches"] == sd["n_launches"] and st["n_candidates"] == 0, (m, kk)
        res.close()
        dense.close()
        hs.close()


def colliders(rng, w, count):
    """`count` words in the hash bucket of w, none equal to w."""
    top = (int(bucket(w)) << 24) | rng.integers(0, 1 << 24, size=count, dtype=np.uint64)
    out = (top * np.uint64(HASH_INV)) & np.uint64(0xFFFFFFFF)
    out = out[out != w].astype(np.uint32)
    assert (bucket(out) == bucket(w)).all()
    return out


def test_hash_collisions(cuda_device, small=False):
    """Patterns whose grams share buckets, and a periodic pattern whose one gram fills many fields at once; text of
    words that collide with a gram's bucket without equalling it, placed where the counted words of an occurrence lie.
    The counters fire on buckets, so such text flags rows; the exact re-check drops every false candidate."""
    rng = np.random.default_rng(24)
    n = 2 * TILE + 333 if small else 5 * TILE + 333
    k = 3
    shared = [int(x) for x in colliders(rng, 0x41424344, 8)]
    pats = [b"".join(w.to_bytes(4, "little") for w in shared) + b"xyz",       # class 0: eight grams, one bucket
            b"abcd" * 9,                                                       # one gram in every field of class 0
            bytes(random_text(rng, 40))]
    total = 0
    for pat in pats:
        m = len(pat)
        Wc = layout(m, k)[0]
        hay = random_text(rng, n)
        words = hay[:n // 4 * 4].view("<u4")
        for t0 in range(7, n // 4 - 2 * Wc, 41):      # fake occurrences of class o0: colliders at their words
            o0 = int(rng.integers(0, 4))
            for i in range(Wc):
                if rng.random() < 0.8:
                    words[t0 + i] = colliders(rng, gram(pat, o0 + 4 * i), 1)[0]
        for s in range(300, n - m - 300, 2039):
            put(hay, s, subs(rng, pat, int(rng.integers(0, k + 2))))
        ends = end_plants(rng, hay, pat, k)
        hs = F.Haystack.from_host(hay)
        marks, raw = search_and_check(hs, pat, hay, k, ends=ends)
        assert marks > 0 and raw > 0
        total += marks
        hs.close()
    assert total > 100


def test_nul_grams_against_the_zeros(cuda_device, small=False):
    """Patterns with runs of NULs, on text that ends in NULs, at lengths around a tile: the zero halo before row 0,
    the buffer's zero padding and the out-of-bounds rows of the last tile hit the table.  The marks still equal the
    restatement, and no match starts before 0 or ends past N."""
    rng = np.random.default_rng(25)
    k = 3
    pats = [bytes(random_text(rng, 10)) + b"\0" * 12 + bytes(random_text(rng, 10)),
            b"\0" * 20 + bytes(random_text(rng, 12)),
            bytes(random_text(rng, 12)) + b"\0" * 20]
    cands = 0
    for n in [TILE + d for d in range(-8, 9)] + [ROW + 3, 2 * TILE - 1]:
        for pat in pats:
            m = len(pat)
            hay = random_text(rng, n)
            hay[-int(rng.integers(5, 40)):] = 0
            put(hay, 0, pat[m // 2:])
            put(hay, n - m + 6, pat[:m - 6])
            seam_plants(rng, hay, pat, k, tile_seams(n))
            hs = F.Haystack.from_host(hay)
            res = hs.search_hamming(pat, k)
            raw = res.triples(F.RAW)
            assert raw == tup(oracle.substitutions(pat, hay, k)), n
            assert all(0 <= s and e <= n for s, e, _ in raw)
            got = res.stats()["n_candidates"]
            assert got == len(hamming_marks(pat, k, hay, 0, 0, n)), (n, pat)
            cands += got
            res.close()
            hs.close()
    assert cands > 0


def test_shards(cuda_device, small=False):
    """Shards whose buffers start at a multiple of 16 that is not one of 128 (their rows are not the whole sequence's
    rows): each shard's count is the restatement of its own buffer clipped to its owned range, and the shards' raw
    lists together are the whole sequence's.  Then one shard at a 40-bit and one at a 44-bit offset."""
    rng = np.random.default_rng(26)
    m, k = 32, 3
    pat = bytes(random_text(rng, m))
    n = 2 * TILE + 4321 if small else 4 * TILE + 4321
    hay = random_text(rng, n)
    for s in range(100, n - 100, 997):
        put(hay, s, subs(rng, pat, int(rng.integers(0, k + 2))))
    for nshards in (2, 3, 7):
        bounds = [0] + [n * i // nshards + int(rng.integers(-64, 64)) for i in range(1, nshards)] + [n]
        h = hay.copy()
        seam_plants(rng, h, pat, k, bounds[1:-1])
        seam_plants(rng, h, pat, k, tile_seams(n))
        whole = tup(oracle.substitutions(pat, h, k))
        union = []
        for i in range(nshards):
            lo, hi = bounds[i], bounds[i + 1]
            blo = max(0, lo - m) // 16 * 16
            if blo % 128 == 0 and blo > 0:
                blo -= 16
            bhi = min(n, hi + m)
            hs = F.Haystack.from_host(h[blo:bhi], buf_lo=blo, global_len=n, own_lo=lo, own_hi=hi)
            res = hs.search_hamming(pat, k)
            assert res.stats()["route"] == HAMMING
            raw = res.triples(F.RAW)
            assert raw == [t for t in whole if lo <= t[0] < hi], (nshards, i)
            assert res.stats()["n_candidates"] == len(hamming_marks(pat, k, h[blo:bhi], blo, lo, hi)), (nshards, i)
            union += raw
            res.close()
            hs.close()
        assert sorted(union) == whole, nshards
    own = [t for t in tup(oracle.substitutions(pat, hay, k)) if 256 <= t[0] < n - 256]
    for shift in ((1 << 40) + 16 * 12345, 1 << 44):
        hs = F.Haystack.from_host(hay, buf_lo=shift, global_len=shift + n + (1 << 20), own_lo=shift + 256,
                                  own_hi=shift + n - 256)
        res = hs.search_hamming(pat, k)
        assert res.triples(F.RAW) == [(s + shift, e + shift, d) for s, e, d in own], shift
        got = res.stats()["n_candidates"]
        assert got == len(hamming_marks(pat, k, hay, shift, shift + 256, shift + n - 256)) > 0, shift
        res.close()
        hs.close()


def test_tiny_work_list_overflows_into_bitmap_mode(cuda_device, small=False):
    """FZB_F_TINY_LIST: the granule work list holds 8 entries and the scan marks far more, so the search runs again
    with the verify kernel sweeping the bitmap; RAW and the marked-granule count stay the same."""
    rng = np.random.default_rng(27)
    m, k = 32, 3
    pat = bytes(random_text(rng, m))
    n = 2 * TILE + 4099
    hay = random_text(rng, n)
    for s in range(200, n - 200, 600):
        put(hay, s, subs(rng, pat, int(rng.integers(0, k + 2))))
    seam_plants(rng, hay, pat, k, tile_seams(n))
    ends = end_plants(rng, hay, pat, k)
    hs = F.Haystack.from_host(hay)
    plain = hs.search_hamming(pat, k)
    check_ends(plain.triples(F.RAW), n, ends)
    res = hs.search_hamming(pat, k, F.F_TINY_LIST)
    assert res.stats()["n_launches"] > plain.stats()["n_launches"]   # the list overflowed: a second attempt ran
    assert res.triples(F.RAW) == plain.triples(F.RAW) == tup(oracle.substitutions(pat, hay, k))
    assert res.stats()["n_candidates"] == plain.stats()["n_candidates"] == len(hamming_marks(pat, k, hay, 0, 0, n)) > 8
    res.close()
    plain.close()
    hs.close()


def test_record_sets(cuda_device, small=False):
    """Records of 0 to m + 1 bytes around row and tile boundaries, and occurrences split by a separator, which the
    counters see as one (the filter reads content only, DESIGN.md section 5.10): each record's list is its single
    search's, and the count is the restatement of the whole joined buffer."""
    rng = np.random.default_rng(28)
    m, k = 32, 3
    pat = bytes(random_text(rng, m))
    recs, pos = [], 0
    for b in (ROW, 4 * ROW, TILE, TILE + 4 * ROW) + (() if small else (2 * TILE, 3 * TILE)):
        fill = b - 60 - pos                          # a long record up to just before the boundary
        assert fill >= 0
        r = random_text(rng, fill)
        for s in range(40, fill - m - 40, 800):
            put(r, s, subs(rng, pat, int(rng.integers(0, k + 2))))
        recs.append(r.tobytes())
        pos += fill + 1
        while pos < b + 60:                          # then short ones across it: 0 to m + 1 bytes
            ln = int(rng.integers(0, m + 2))
            rec = subs(rng, pat, int(rng.integers(0, k + 2)))
            rec = (rec + b"!")[:ln] if rng.random() < 0.5 else (b"!" + rec)[m + 1 - ln:]
            recs.append(rec)
            pos += len(rec) + 1
        cut = int(rng.integers(4, m - 4))             # an occurrence split by the separator after this record
        recs.append(bytes(random_text(rng, 50)) + pat[:cut])
        recs.append(pat[cut:] + bytes(random_text(rng, 50)))
        pos += len(recs[-1]) + len(recs[-2]) + 2
    buf = b"\0".join(recs) + b"\0"
    off = np.zeros(len(recs) + 1, dtype=np.uint64)
    off[1:] = np.cumsum([len(r) + 1 for r in recs])
    hs = F.Haystack.from_host(buf)
    hs.set_records(off)
    res = hs.search_hamming(pat, k)
    assert res.stats()["route"] == HAMMING
    raw = res.triples(F.RAW)
    assert res.triples(F.FINAL) == raw
    assert res.stats()["n_candidates"] == len(hamming_marks(pat, k, buf, 0, 0, len(buf))) > 0
    res.close()
    single = F.Haystack.alloc(max(len(r) for r in recs))
    got = 0
    for i, r in enumerate(recs):
        b = int(off[i])
        mine = [(s - b, e - b, d) for s, e, d in raw if b <= s < int(off[i + 1])]
        single.upload(r)
        one = single.search_hamming(pat, k)
        assert mine == one.triples(F.RAW) == tup(oracle.substitutions(pat, r, k)), (i, len(r))
        one.close()
        got += len(mine)
    assert got == len(raw) > 0
    single.close()
    hs.close()


def test_reupload_shorter_contents(cuda_device, small=False):
    """fzb_haystack_upload of shorter contents into a handle that held text full of occurrences: the padding after the
    new end is zeroed again and the rows past it read as zeros, so the restatement with zeros holds on the second
    search too."""
    rng = np.random.default_rng(29)
    m, k = 32, 3
    pat = bytes(random_text(rng, m))
    n0 = 3 * TILE + 100
    full = np.frombuffer(pat * (n0 // m + 1), dtype=np.uint8)[:n0].copy()
    hs = F.Haystack.from_host(full)
    search_and_check(hs, pat, full, k)
    for n in (TILE + 77, ROW - 5, 2 * TILE - 16, 5):
        hay = random_text(rng, n)
        ends = end_plants(rng, hay, pat, k)
        hs.upload(hay)
        if n >= m:
            search_and_check(hs, pat, hay, k, ends=ends)
        else:
            res = hs.search_hamming(pat, k)
            assert res.triples(F.RAW) == [] and res.stats()["n_candidates"] == len(hamming_marks(pat, k, hay, 0, 0, n))
            res.close()
    hs.close()
