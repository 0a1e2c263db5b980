"""k_filter_sampled, the scan of the benchmarked search, at the geometry of its shared-memory ring: 32 KiB tiles
copied into stages in turn, the last tile partial, the persistent grid striding over them.

What the scan decides is the set of marked granules, and stats()["n_candidates"] counts them.  The tests restate
that set in numpy -- the 4-byte-aligned words of the buffer (counted from its first byte, the zero padding up to the
next multiple of 16 included) that equal one of the pattern's m - 3 grams, each marking the granules of the anchors
[g - (m + k - 4), g + (m - L + k)] clipped to the owned range -- and compare the count; the raw stream (in generation
order, with its anchors) and the final list are compared with the oracle."""
import numpy as np
import pytest

import oracle
from corpus import ASCII
from fuzzysearch_b200 import _native as F
from parity import tup

pytestmark = pytest.mark.gpu

SAMPLED = "ngrams/sampled-filter"
STAGE = 32768                 # bytes per ring stage = per tile (kernels.cuh: kScanStageBytes)
GRID_PASS = 2 * 132 * STAGE   # tiles of one pass of the grid on an H100: two CTAs per SM
EMU_PASS = 4 * STAGE          # the emulated device: 2 SMs, 2 CTAs per SM


def random_text(rng, n, alphabet=ASCII):
    alpha = np.frombuffer(alphabet, dtype=np.uint8)
    return alpha[rng.integers(0, len(alpha), size=n)].copy()


def variant(rng, pat, k):
    """P with up to k random edits (substitution, deletion or insertion)."""
    v = bytearray(pat)
    for _ in range(int(rng.integers(0, k + 1))):
        i = int(rng.integers(1, len(v) - 1))
        op = int(rng.integers(0, 3))
        if op == 0:
            v[i] = (v[i] + 1) % 256
        elif op == 1:
            del v[i]
        else:
            v.insert(i, v[i - 1])
    return bytes(v)


def put(hay, pos, v):
    v = np.frombuffer(bytes(v), dtype=np.uint8)[:max(0, len(hay) - pos)]
    hay[pos:pos + len(v)] = v


def seam_plants(rng, hay, pat, k, lo=0):
    """Occurrences ending in the last 16 bytes of a stage, crossing a seam, and in the first 16 bytes of the next,
    at every stage seam of the buffer (buffer offsets, the buffer starting at hay[lo])."""
    m = len(pat)
    for b in range(STAGE, len(hay) - lo, STAGE):
        for s in (b - m - int(rng.integers(0, 12)), b - m // 2, b + int(rng.integers(0, 12))):
            put(hay, lo + s, variant(rng, pat, k))


def end_plants(rng, hay, pat, k):
    """Occurrences in the last, partial stage: one ending at the last byte, one a few bytes before it, and a pattern
    prefix cut off by the end."""
    n, m = len(hay), len(pat)
    put(hay, n - m - 7, variant(rng, pat, k))
    put(hay, n - m, pat)
    put(hay, n - m // 2, pat)


def marked_granules(pat, k, buf, buf_lo, own_lo, own_hi):
    """The granules k_filter_sampled marks on the buffer `buf` (its bytes up to the next multiple of 16 included)."""
    m = len(pat)
    L = m // (k + 1)
    nv = (len(buf) + 15) // 16 * 16
    b = np.zeros(nv, dtype=np.uint8)
    b[:len(buf)] = buf
    words = b.view("<u4")
    grams = np.array([int.from_bytes(pat[o:o + 4], "little") for o in range(m - 3)], dtype=np.uint32)
    g = buf_lo + 4 * np.nonzero(np.isin(words, grams))[0].astype(np.int64)
    lo = np.maximum(g - (m + k - 4), own_lo)
    hi = np.minimum(g + (m - L + k), own_hi - 1)
    keep = lo <= hi
    g0, g1 = (lo[keep] - buf_lo) >> 6, (hi[keep] - buf_lo) >> 6
    out = set()
    for d in range(int((g1 - g0).max()) + 1 if g0.size else 0):
        out.update(int(x) for x in (g0 + d)[g0 + d <= g1])
    return out


def anchored(res):
    s, e, d, ng, ix = res.arrays(F.RAW, anchors=True)
    return list(zip(ng.tolist(), ix.tolist(), s.tolist(), e.tolist(), d.tolist()))


def oracle_anchored(pat, hay, k):
    raw, ng, ix = oracle.levenshtein_ngrams_raw(pat, hay, k, with_anchor=True)
    return [(int(a), int(b)) + t for a, b, t in zip(ng, ix, tup(raw))], raw


def search_and_check(hs, pat, hay, k, flags=0):
    """One whole-sequence search: raw stream with anchors and final list against the oracle, the candidate count
    against the restated marks -> the number of raw records."""
    res = hs.search_levenshtein(pat, k, F.F_FORCE_SAMPLED | flags)
    st = res.stats()
    assert st["route"] == SAMPLED
    want, raw = oracle_anchored(pat, hay, k)
    assert anchored(res) == want, len(hay)
    assert res.triples(F.FINAL) == tup(oracle.consolidate(raw)), len(hay)
    assert st["n_candidates"] == len(marked_granules(pat, k, hay, 0, 0, len(hay))), len(hay)
    res.close()
    return len(want)


def lengths_around(bases):
    return [b + d for b in bases for d in range(-8, 8)]   # every residue mod 16 around each base


def test_buffer_lengths_around_stages_and_the_grid_pass(cuda_device, small=False):
    """Buffers of every length mod 16 around 1, 2 and 3 stages and around one pass of the grid, with occurrences at
    every stage seam and in the last, partial stage."""
    rng = np.random.default_rng(5)
    m, k = 20, 2
    pat = bytes(random_text(rng, m))
    grid_pass = EMU_PASS if small else GRID_PASS
    base = random_text(rng, grid_pass + 64)
    seam_plants(rng, base, pat, k)
    total = 0
    for n in lengths_around([STAGE, 2 * STAGE, 3 * STAGE, grid_pass]):
        hay = base[:n].copy()
        end_plants(rng, hay, pat, k)
        hs = F.Haystack.from_host(hay)
        total += search_and_check(hs, pat, hay, k)
        hs.close()
    assert total >= 2 * 64


def test_pattern_with_nul_bytes_against_the_zero_padding(cuda_device, small=False):
    """A pattern whose grams hold NUL bytes: aligned words reaching into the zero padding after the last byte (up to
    the next multiple of 16) equal such grams, and the scan marks them exactly as it would marks of real bytes."""
    rng = np.random.default_rng(6)
    k = 2
    pat = bytes(random_text(rng, 13)) + b"\0" * 7
    n0 = STAGE if small else 3 * STAGE
    cands = 0
    for n in range(n0 + 1, n0 + 17):
        hay = random_text(rng, n)
        hay[-3:] = 0                      # the last bytes are NULs too: words across the end equal grams
        put(hay, n - 30, variant(rng, pat[:-3], k))
        seam_plants(rng, hay, pat, k)
        hs = F.Haystack.from_host(hay)
        res = hs.search_levenshtein(pat, k, F.F_FORCE_SAMPLED)
        assert anchored(res) == oracle_anchored(pat, hay, k)[0], n
        got = res.stats()["n_candidates"]
        assert got == len(marked_granules(pat, k, hay, 0, 0, n)), n
        cands += got
        res.close()
        hs.close()
    assert cands > 0


def test_shards_at_offsets(cuda_device, small=False):
    """Shards of one sequence whose buffers start at buf_lo != 0 (halo included, multiples of 16), and a shard whose
    buffer starts at a 64-bit offset: every shard's marks are its own buffer's words clipped to its owned range, and
    the shards' raw streams together are the whole sequence's."""
    rng = np.random.default_rng(7)
    m, k = 20, 2
    pat = bytes(random_text(rng, m))
    n = 3 * STAGE + 4321
    hay = random_text(rng, n)
    seam_plants(rng, hay, pat, k)
    for s in range(100, n - 100, 997):
        put(hay, s, variant(rng, pat, k))
    want = sorted(tup(oracle.levenshtein_ngrams_raw(pat, hay, k)))
    bounds = [0, STAGE - 40, 2 * STAGE + 13, n]
    halo = m + k
    union = []
    for i in range(len(bounds) - 1):
        lo, hi = bounds[i], bounds[i + 1]
        blo = max(0, lo - halo) // 16 * 16
        bhi = min(n, hi + halo)
        hs = F.Haystack.from_host(hay[blo:bhi], buf_lo=blo, global_len=n, own_lo=lo, own_hi=hi)
        res = hs.search_levenshtein(pat, k, F.F_FORCE_SAMPLED | F.F_NO_FINAL)
        assert res.stats()["route"] == SAMPLED
        assert res.stats()["n_candidates"] == len(marked_granules(pat, k, hay[blo:bhi], blo, lo, hi)), i
        union += res.triples(F.RAW)
        res.close()
        hs.close()
    assert sorted(union) == want
    shift = (1 << 40) + 16 * 12345
    hs = F.Haystack.from_host(hay, buf_lo=shift, global_len=shift + n + (1 << 20), own_lo=shift + 256,
                              own_hi=shift + n - 256)
    res = hs.search_levenshtein(pat, k, F.F_FORCE_SAMPLED)
    assert res.stats()["n_candidates"] == len(marked_granules(pat, k, hay, shift, shift + 256, shift + n - 256))
    own = sorted((s + shift, e + shift, d) for s, e, d in tup(oracle.levenshtein_ngrams_raw(pat, hay, k))
                 if 256 <= s and e <= n - 256)
    assert [t for t in sorted(res.triples(F.RAW)) if t in set(own)] == own
    res.close()
    hs.close()


def test_exact_search_windows(cuda_device, small=False):
    """search_exact over windows: a view of the resident buffer from a 128-byte boundary a halo before `start` to
    `end`, owning [start, end); the scan reads the view's bytes up to the next multiple of 16, which past `end` are
    the resident sequence's own."""
    rng = np.random.default_rng(8)
    m = 12
    pat = bytes(random_text(rng, m))
    n = 3 * STAGE + 777
    hay = random_text(rng, n)
    seam_plants(rng, hay, pat, 0)
    for s in range(50, n - 50, 1499):
        put(hay, s, pat)
    hs = F.Haystack.from_host(hay)
    padded = np.concatenate([hay, np.zeros(256, dtype=np.uint8)])
    halo = (m + 127) // 128 * 128 + 128
    for start, end in ((0, n), (1, n - 1), (STAGE - 5, 2 * STAGE + 9), (1000, 3 * STAGE + 3), (STAGE + 17, n)):
        res = hs.search_exact(pat, F.F_FORCE_SAMPLED, start=start, end=end)
        assert [s for s, _, _ in res.triples(F.RAW)] == oracle.search_exact(pat, bytes(hay), start, end), (start, end)
        vlo = (start - halo if start > halo else 0) // 128 * 128
        view = padded[vlo:end]
        nv = (len(view) + 15) // 16 * 16
        got = res.stats()["n_candidates"]
        assert got == len(marked_granules(pat, 0, padded[vlo:vlo + nv], vlo, start, end)), (start, end)
        res.close()
    hs.close()


def test_tiny_work_list_overflows_into_bitmap_mode(cuda_device, small=False):
    """FZB_F_TINY_LIST: the granule work list holds 8 entries, the scan marks far more, and the search is repeated
    with the verify kernel sweeping the bitmap; results and the marked-granule count stay the same."""
    rng = np.random.default_rng(9)
    m, k = 20, 2
    pat = bytes(random_text(rng, m))
    n = 2 * STAGE + 4099
    hay = random_text(rng, n)
    seam_plants(rng, hay, pat, k)
    for s in range(200, n - 200, 1200):
        put(hay, s, variant(rng, pat, k))
    end_plants(rng, hay, pat, k)
    hs = F.Haystack.from_host(hay)
    res = hs.search_levenshtein(pat, k, F.F_FORCE_SAMPLED | F.F_TINY_LIST)
    assert res.stats()["n_launches"] > 3   # the list overflowed: a second attempt ran
    assert anchored(res) == oracle_anchored(pat, hay, k)[0]
    assert res.stats()["n_candidates"] == len(marked_granules(pat, k, hay, 0, 0, n)) > 8
    res.close()
    hs.close()
