"""fzb_nearest_distance / fzb_nearest_per_record, find_nearest_matches / nearest_distance(_in_each) (DESIGN.md section
5.14): the nearest match without a distance limit.  Every case compares `dist`, `n_ends`, `first_end` and, per record,
`(dist, end)` exactly with `nearest_E`, a numpy restatement of Sellers' table that knows nothing of bit vectors,
segments or warm-ups (tests/test_host_nearest.py checks it against a plain triple loop and the oracle).  `small` keeps
the sizes the CPU emulator replays (tests/test_emu_nearest.py)."""
import numpy as np
import pytest

from fuzzysearch_b200 import (DeviceSequence, DeviceSequenceSet, NearestDistances, _native as F, find_near_matches,
                              find_nearest_matches, nearest_distance, nearest_distance_in_each)
from test_gpu_records import joined, rand

pytestmark = pytest.mark.gpu

THREADS, MIN_SEG, MAX_SEG = 256, 512, 4096  # nearest_kernels.cuh
M_SIZES = (1, 2, 31, 32, 33, 63, 64, 65, 128, 255)


def nearest_E(P, S, block=1 << 20):
    """E[..., e] = min over s <= e of lev(P, S[..., s:e]) for e in 0..n, for one text or a stack of equally long
    texts.  Row by row over the pattern; inside a row D[i][j] = min(t[j], D[i][j-1] + 1) is
    minimum.accumulate(t - arange) + arange, taken in column blocks that hand the running minimum on."""
    P = np.frombuffer(bytes(P), dtype=np.uint8)
    S = np.frombuffer(S, dtype=np.uint8) if isinstance(S, (bytes, bytearray)) else np.asarray(S, dtype=np.uint8)
    n = S.shape[-1]
    prev = np.zeros(S.shape[:-1] + (n + 1,), dtype=np.int16)  # D[0][j] = 0: a match may start anywhere
    for i in range(1, len(P) + 1):
        cur = np.empty_like(prev)
        cur[..., 0] = i
        carry = np.full(S.shape[:-1] + (1,), i, dtype=np.int32)  # D[i][j0 - 1] - (j0 - 1) of the block before
        for j0 in range(1, n + 1, block):
            j1 = min(j0 + block, n + 1)
            ar = np.arange(j0, j1, dtype=np.int32)
            t = np.minimum(prev[..., j0:j1].astype(np.int32) + 1,
                           prev[..., j0 - 1:j1 - 1] + (S[..., j0 - 1:j1 - 1] != P[i - 1]))
            acc = np.minimum(np.minimum.accumulate(t - ar, axis=-1), carry)
            carry = acc[..., -1:]
            cur[..., j0:j1] = acc + ar
        prev = cur
    return prev


def nearest(P, S):
    """-> (d*, n_ends, first_end) of one text"""
    E = nearest_E(P, S)
    d = int(E.min())
    at = np.flatnonzero(E == d)
    return d, int(at.size), int(at[0])


def nearest_rows(P, rows):
    """-> (dist, end) arrays for a stack of equally long texts"""
    E = nearest_E(P, rows)
    return E.min(axis=-1).astype(np.int32), E.argmin(axis=-1).astype(np.int64)


def segmented(P, S, seg, warm):
    """The per-segment scheme transcribed on the host: every segment of `seg` bytes is scanned from a fresh column
    started `warm` bytes before it, and only the ends inside the segment count."""
    m, n = len(P), len(S)
    best = (m, 1, 0)  # the end position 0
    for a in range(0, n, seg):
        w = max(a - warm, 0)
        E = nearest_E(P, S[w:min(a + seg, n)])[a - w + 1:]
        d = int(E.min())
        at = np.flatnonzero(E == d)
        if d < best[0]:
            best = (d, int(at.size), a + 1 + int(at[0]))
        elif d == best[0]:
            best = (d, best[1] + int(at.size), min(best[2], a + 1 + int(at[0])))
    return best


def seg_of(n, sms):
    """nearest_scan's choice of the bytes per thread (api.cu)"""
    return min(MAX_SEG, max(MIN_SEG, (n // (sms * 1024) + 1 + 15) // 16 * 16))


def seam_cases(rng, m, seam, offsets):
    """Binary texts of 2 * seam bytes, all 'b' but for one stretched copy of a random pattern that ends at seam + o,
    for every o: behind four symbols in ten (every third case: nine in ten, nearly 2m long) stands the other letter,
    so the best alignment reaches far behind the seam."""
    for o in offsets:
        P = rand(rng, b"ab", m)
        stretch = 0.9 if o % 3 == 0 else 0.4
        grown = b"".join(bytes([c]) + (bytes([c ^ 3]) if rng.random() < stretch else b"") for c in P)  # 'a' ^ 3 == 'b'
        text = bytearray(b"b" * (2 * seam))
        text[seam + o - len(grown):seam + o] = grown
        yield P, bytes(text)


def check_handle(hs, P, S, ctx=()):
    d, n_ends, first, st = hs.nearest_distance(P)
    assert (d, n_ends, first) == nearest(P, S), ctx + (len(P), len(S))
    assert st["route"] == "nearest/bit-vector-scan" and st["bytes_scanned"] == len(S)
    return d


def test_pattern_sizes_and_short_texts(cuda_device, small=False):
    rng = np.random.default_rng(11)
    hs = F.Haystack.alloc(1 << 16, device=cuda_device)
    for m in M_SIZES:
        for alphabet in (b"ab", b"ACGT", bytes(range(256))):
            P = rand(rng, alphabet, m)
            for n in sorted({0, 1, m - 1, 2 * m - 1, 2 * m + 1, 3 * m + 7, 700}):
                if small and n == 700 and m not in (32, 33, 255):
                    continue
                S = bytearray(rand(rng, alphabet, n))
                if n >= m and rng.random() < 0.5:
                    S[n - m:] = P  # an exact occurrence closing the text
                hs.upload(bytes(S))
                check_handle(hs, P, bytes(S), (alphabet[:4],))
    hs.close()


def test_lengths_around_segments_tiles_and_grid_passes(cuda_device, small=False):
    """Every length mod 16 around one segment and one tile; whole grid passes (the grid of the emulator is small
    enough for three of them, the device takes more than one with a longer segment)."""
    rng = np.random.default_rng(12)
    tile = THREADS * MIN_SEG
    lengths = [MIN_SEG + d for d in range(-17, 18)] + [tile + d for d in range(-17, 18, 1 if not small else 5)]
    if small:
        passes = 2 * 4 * tile  # FZB_EMU_SMS=2, four CTAs per SM
        lengths += [passes - 1, 2 * passes + 3, 3 * passes - 16 + 5]
    base = rand(rng, b"ACGT", max(lengths))
    hs = F.Haystack.alloc(max(lengths), device=cuda_device)
    for m, P in ((20, rand(rng, b"ACGT", 20)), (40, rand(rng, b"ACGT", 40))):
        for n in lengths if m == 20 else lengths[::7]:
            S = bytearray(base[:n])
            S[max(n - 2 * m, 0):] = rand(rng, b"ACGT", min(2 * m, n))
            if n >= m:
                S[n - m:] = P[:m - 1] + b"A"  # the best end is the last position or close to it
            hs.upload(bytes(S))
            check_handle(hs, P, bytes(S))
    hs.close()
    if not small:  # more than one grid pass on the device: 160 MB at the segment length the host then picks
        n = 160_000_003
        S = bytearray(rand(rng, b"ACGT", n))
        P = b"GATTACAGGT"
        S[n - 10:] = P
        S[77_000_000:77_000_010] = P
        hs = F.Haystack.from_host(bytes(S), device=cuda_device)
        check_handle(hs, P, bytes(S))
        hs.close()


def test_best_occurrence_at_every_offset_around_the_seams(cuda_device, small=False):
    """... and a warm-up of only m bytes, transcribed on the host, gets one of these cases wrong (few of them do: the
    seed is one whose cases include such a text at either step)."""
    rng = np.random.default_rng(28)
    tile = THREADS * MIN_SEG
    short_warmup_fails = 0
    for m, seam, offsets in ((24, MIN_SEG, range(-4, 2 * 24 + 6, 1 if not small else 3)),
                             (33, tile, range(-4, 2 * 33 + 6, 1 if not small else 9))):
        hs = F.Haystack.alloc(2 * seam, device=cuda_device)
        for P, S in seam_cases(rng, m, seam, offsets):
            hs.upload(S)
            check_handle(hs, P, S)
            if seam == MIN_SEG:
                assert segmented(P, S, MIN_SEG, 2 * m) == nearest(P, S)
                short_warmup_fails += segmented(P, S, MIN_SEG, m) != nearest(P, S)
        hs.close()
    assert short_warmup_fails > 0


def test_ties_extremes_and_byte_values(cuda_device):
    rng = np.random.default_rng(14)
    hs = F.Haystack.alloc(1 << 16, device=cuda_device)
    cases = [(b"GATTACA", b"xxGATTACAxxGATTACAxxxGATTACA"),            # d* = 0, three ends
             (b"GATTACA", b"xxGATTCAxxGATTTACAxx"),                     # ties at d* = 1
             (b"abc", b"xyzxyzxyz" * 100),                              # d* = m: no pattern symbol in the text
             (b"\0\0\0\0", b"abcd" * 33),                               # a NUL pattern against the zero padding
             (b"\0\0\0", b"ab\0"), (b"\0" * 40, b"\0" * 39), (b"\0" * 70, b"x" * 127 + b"\0"),
             (bytes(range(128, 160)), rand(rng, bytes(range(120, 170)), 3000)),
             (bytes(range(200, 256)) + bytes(range(9)), bytes(range(256)) * 9),
             (bytes(range(256))[:255], bytes(reversed(range(256))) * 3 + bytes(range(256)))]
    for P, S in cases:
        hs.upload(S)
        check_handle(hs, P, S)
    hs.upload(b"xyzxyzxyz")
    assert hs.nearest_distance(b"abc")[:3] == (3, 10, 0)
    hs.close()


def test_reupload_and_searches_around_the_call(cuda_device):
    rng = np.random.default_rng(15)
    P = rand(rng, b"ACGT", 24)
    texts = []
    for n in (5000, 300, 70000):
        S = bytearray(rand(rng, b"ACGT", n))
        S[n // 2:n // 2 + 24] = P[:11] + b"A" + P[12:]
        texts.append(bytes(S))
    hs = F.Haystack.alloc(70000, device=cuda_device)
    for S in texts:
        hs.upload(S)
        before = hs.search_levenshtein(P, 3)
        b_raw, b_fin = before.triples(F.RAW), before.triples(F.FINAL)
        held = hs.search_levenshtein(P, 2)  # its raw records stay on the device across the call
        d = check_handle(hs, P, S)
        assert d <= 1
        h_raw = held.triples(F.RAW)
        after = hs.search_levenshtein(P, 3)
        assert (after.triples(F.RAW), after.triples(F.FINAL)) == (b_raw, b_fin)
        again = hs.search_levenshtein(P, 2)
        assert again.triples(F.RAW) == h_raw
        for r in (before, held, after, again):
            r.close()
    hs.close()


def check_records(hs, P, recs, ctx=()):
    buf, off = joined(recs)
    hs.upload(buf)
    hs.set_records(off)
    dist, end, st = hs.nearest_per_record(P)
    assert dist.dtype == np.int32 and end.dtype == np.int64 and len(dist) == len(recs)
    exp = [nearest(P, r) for r in recs]
    assert dist.tolist() == [e[0] for e in exp], ctx
    assert end.tolist() == [e[2] for e in exp], ctx
    assert st["route"] == "nearest/bit-vector-scan"
    return dist, end


def test_record_sets(cuda_device, small=False):
    rng = np.random.default_rng(16)
    hs = F.Haystack.alloc(12 << 20, device=cuda_device)
    P = b"GATTACAGATC"
    lengths = list(range(0, 301))
    for order in ("up", "down", "shuffled"):
        ls = lengths if order == "up" else lengths[::-1] if order == "down" else list(rng.permutation(lengths))
        recs = [rand(rng, b"ACGT", int(n)) for n in ls]
        check_records(hs, P, recs, (order,))
    # separators that equal pattern bytes: a NUL pattern must not match across or on them
    recs = [b"", b"\0", b"ab", b"\0\0", b"", b"a\0", b"\0a", b"\0" * 5, b""]
    for Pz in (b"\0", b"\0\0", b"\0\0\0", b"a\0\0a", b"\0" * 40):
        check_records(hs, Pz, recs, (Pz,))
    # one long record among short ones, first and last records holding the best matches at their very edges
    big = (1 << 20) if small else (9 << 20)
    for m in (11, 40, 70):
        Pm = rand(rng, b"ACGT", m)
        long_rec = bytearray(rand(rng, b"ACGT", big))
        long_rec[big - m:] = Pm
        long_rec[:m] = Pm[1:] + b"A"
        recs = [Pm] + [rand(rng, b"ACGT", 150) for _ in range(40)] + [bytes(long_rec)] + \
               [rand(rng, b"ACGT", 150) for _ in range(40)] + [Pm[:-1]]
        dist, end = check_records(hs, Pm, recs, (m,))
        assert (dist[0], end[0]) == (0, m) and dist[41] == 0 and (dist[-1], end[-1]) == (1, m - 1)
        # per-record answers are those of each record alone, through the whole-sequence entry point
        hs.set_records(None)
        for r in (0, 7, 41, len(recs) - 1):
            hs.upload(recs[r])
            assert hs.nearest_distance(Pm)[::2] == (int(dist[r]), int(end[r]))
    hs.close()


def test_one_million_reads(cuda_device, small=False):
    rng = np.random.default_rng(17)
    count, n = (3000, 150) if small else (1_000_000, 150)
    P = b"AGATCGGAAGAGCACACGTCTGAACTCCAGTCA"[:25]
    rows = np.frombuffer(rand(rng, b"ACGT", count * n), dtype=np.uint8).reshape(count, n).copy()
    at = rng.integers(0, n - 25, size=count)
    for r in range(0, count, 3):  # a third of the reads carry the adapter with up to three substitutions
        v = np.frombuffer(P, dtype=np.uint8).copy()
        v[rng.integers(0, 25, size=int(rng.integers(0, 4)))] = ord("N")
        rows[r, at[r]:at[r] + 25] = v
    reads = [bytes(r) for r in rows]
    got = nearest_distance_in_each(P, reads)
    assert isinstance(got, NearestDistances) and len(got) == count
    exp_d, exp_e = [], []
    for lo in range(0, count, 100_000):
        d, e = nearest_rows(P, rows[lo:lo + 100_000])
        exp_d.append(d)
        exp_e.append(e)
    assert np.array_equal(got.dist, np.concatenate(exp_d)) and np.array_equal(got.end, np.concatenate(exp_e))
    assert got[0] == (int(got.dist[0]), int(got.end[0]))


def test_public_api(cuda_device, small=False):
    rng = np.random.default_rng(18)
    n = 20000 if small else 300000
    S = bytearray(rand(rng, b"ACGT", n))
    P = rand(rng, b"ACGT", 30)
    # planted at distance 0 / 2 (n-gram route: 30 // 3 >= 3) / none (d* lands on the LP route: 12 // (d* + 1) < 3)
    for planted, pat in ((P, P), (P[:7] + b"T" + P[8:19] + P[20:], P), (b"", rand(rng, b"ACGT", 12))):
        S2 = bytes(S[:n // 2] + planted + S[n // 2:])
        d = nearest_distance(pat, S2)
        assert d == nearest(pat, S2)[0]
        exp = find_near_matches(pat, S2, max_l_dist=d)
        assert exp and find_nearest_matches(pat, S2) == exp
        assert find_nearest_matches(pat, S2, max_l_dist=d) == exp
        assert find_nearest_matches(pat, S2, max_l_dist=d + 3) == exp
        if d:
            assert find_nearest_matches(pat, S2, max_l_dist=d - 1) == []
            assert find_near_matches(pat, S2, max_l_dist=d - 1) == []
        ds = DeviceSequence(S2, device=cuda_device)
        assert find_nearest_matches(pat, ds) == exp and nearest_distance(pat, ds) == d
        assert find_nearest_matches(pat, ds) == exp
        ds.close()
    # str (latin-1, general Unicode) and lists of items
    for pat, seq in (("café au lait", "xx cafe au lait, café ou lait xx" * 3),
                     ("ΑΒΓΔΕΖΗΘ", "αβγδ ΑΒΓΕΖΗΘ \U0001F600 ΑΒΓΔΕΖΗΘ"[:-2] + "λ"),
                     ("abc", "ΑΒΓ" * 10),
                     (["x", 3, "y", 4.5], [1, "x", 3, "z", 4.5, (), "x", "y"] * 4)):
        d = nearest_distance(pat, seq)
        exp = find_near_matches(pat, seq, max_l_dist=d)
        assert exp and find_nearest_matches(pat, seq) == exp, pat
        assert d == 0 or find_near_matches(pat, seq, max_l_dist=d - 1) == []
        if isinstance(seq, str):
            ds = DeviceSequence(seq, device=cuda_device)
            assert find_nearest_matches(pat, ds) == exp and find_nearest_matches(pat, ds, max_l_dist=d) == exp
            ds.close()
    # sets: lists, str, resident sets reused across patterns
    recs = [rand(rng, b"ACGT", int(k)) for k in rng.integers(0, 200, size=50)] + [b"", P]
    got = nearest_distance_in_each(P, recs)
    assert got.dist.tolist() == [nearest_distance(P, r) for r in recs]
    assert got[len(recs) - 2] == (30, 0) and got[len(recs) - 1] == (0, 30)
    seqset = DeviceSequenceSet(recs, device=cuda_device)
    for pat in (P, P[:9], b"N" * 5):
        got = nearest_distance_in_each(pat, seqset)
        exp = [nearest(pat, r) for r in recs]
        assert got.dist.tolist() == [e[0] for e in exp] and got.end.tolist() == [e[2] for e in exp]
    seqset.close()
    words = ["naïve", "", "ΑΒΓ naive", "nave", "\U0001F600naïv"]
    got = nearest_distance_in_each("naïve", words)
    assert got.dist.tolist() == [0, 5, 1, 1, 1] and got.end.tolist() == [5, 0, 9, 4, 5]
    assert len(nearest_distance_in_each(P, [])) == 0
    for call in (lambda: nearest_distance(b"", b"abc"), lambda: find_nearest_matches(b"", b"abc"),
                 lambda: nearest_distance_in_each(b"", [b"abc"]), lambda: find_nearest_matches(b"a", b"abc", -1)):
        with pytest.raises(ValueError):
            call()


def test_refusals_leave_the_handle_usable(cuda_device):
    rng = np.random.default_rng(19)
    S = rand(rng, b"ACGT", 5000)
    P = S[1000:1020]
    hs = F.Haystack.from_host(S, device=cuda_device)
    good = hs.nearest_distance(P)[:3]
    assert good == nearest(P, S)

    def still_good():
        assert hs.nearest_distance(P)[:3] == good
        res = hs.search_levenshtein(P, 1)
        assert (1000, 1020, 0) in res.triples(F.FINAL)
        res.close()

    with pytest.raises(F.UnsupportedError):
        hs.nearest_distance(P, flags=16)
    with pytest.raises(ValueError):
        hs.nearest_distance(b"")
    with pytest.raises(F.UnsupportedError):
        hs.nearest_distance(b"A" * 256)
    with pytest.raises(ValueError):
        hs.nearest_per_record(P)  # no record set
    still_good()
    hs.set_records(np.array([0, 2500, 5000], dtype=np.uint64))
    with pytest.raises(F.UnsupportedError):
        hs.nearest_distance(P)  # a record set, as has_near_match refuses it
    with pytest.raises(F.UnsupportedError):
        hs.nearest_per_record(P, flags=1)
    with pytest.raises(ValueError):
        hs.nearest_per_record(b"")
    dist, end, _ = hs.nearest_per_record(P)
    assert (dist.tolist(), end.tolist()) == ([0, nearest(P, S[2500:4999])[0]], [1020, nearest(P, S[2500:4999])[2]])
    hs.set_records(None)
    still_good()
    hs.close()
    # a shard and a handle in a world
    shard = F.Haystack.from_host(S[:4096], device=cuda_device, buf_lo=0, global_len=5000, own_lo=0, own_hi=2048)
    with pytest.raises(F.UnsupportedError):
        shard.nearest_distance(P)
    res = shard.search_levenshtein(P, 0)
    assert res.triples(F.RAW) == [(1000, 1020, 0)]
    res.close()
    shard.close()
    world = F.Haystack.from_host(S, device=cuda_device)
    F.comm_init_local([world])
    with pytest.raises(F.UnsupportedError):
        world.nearest_distance(P)
    world.close()
