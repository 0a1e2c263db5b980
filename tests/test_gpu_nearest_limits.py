"""The nearest scans and the per-record reductions at the limits of their packed fields (DESIGN.md sections 5.13-5.16):
ends and counts past 2^32 on one sequence, records of 2^32 - 1 and 2^31 - 1 bytes, segment lengths between the
shortest and the longest, 65 535 patterns.  Every case covers Levenshtein and substitutions only.

The inputs past 2^32 are never built on the host.  The buffer is filled on the device with BACKGROUND bytes, which
no pattern here holds, and pattern-alphabet regions of a few KB are written into it.  `windowed` then restates the
answer exactly from read-backs around the regions: E(e) depends only on S[e - 2m : e] (section 5.14) and H(e) only
on S[e - m : e], so an end whose window holds background bytes alone scores m, and every other end is restated by
`nearest_E` / `hamming_H` over the region read back with 2m bytes on either side.  The 65 535 patterns are mostly
made of bytes absent from the text; their rows are known in closed form, and the live ones are restated.  `small`
keeps the sizes the CPU emulator replays (tests/test_emu_nearest_limits.py)."""
import numpy as np
import pytest

import oracle
from conftest import needs_real_gpu
from fuzzysearch_b200 import _native as F
from test_gpu_best_match import NAMES, reduce_lists
from test_gpu_nearest import MAX_SEG, THREADS, nearest, nearest_E, seam_cases, seg_of
from test_gpu_nearest_batch import reduce_rows as lev_reduce_rows, sm_count, warp_seg
from test_gpu_nearest_hamming import NONE32, NONE64, SUB, hamming, hamming_H, reduce_rows as ham_reduce_rows
from test_gpu_records import joined, rand

pytestmark = pytest.mark.gpu

BACKGROUND = b"wxyz"  # no pattern of this file holds one of these bytes
METRICS = (0, SUB)
G32, G31 = 1 << 32, 1 << 31


def grid_of(n, m, sms):
    """near_geometry's CTAs for a pattern of m symbols (api.cu)"""
    tile = THREADS * seg_of(n, sms)
    return min(-(-n // tile), sms * (4 if m <= 32 else 3 if m <= 64 else 2), 1024)


def big_n(sms):
    """A sequence past 2^32 + 2^20 long enough that the scans of every word class (m <= 32, m <= 64, m <= 255) start
    a grid pass above 2^32"""
    passes = [grid_of(G32, m, sms) * THREADS * MAX_SEG for m in (24, 40, 100)]
    return max([G32] + [-(-(G32 + 1) // p) * p for p in passes]) + (1 << 20) + 7


def column(P, T, flags):
    """(score, end) of every end E / H defines in the text T (or a stack of equally long texts), ends relative to
    T's start"""
    if flags & SUB:
        H = hamming_H(P, T).astype(np.int64)
        return H, np.arange(len(P), len(P) + H.shape[-1])
    E = nearest_E(P, T)
    return E.astype(np.int64), np.arange(E.shape[-1])


def windowed(read, P, flags, lo, hi, regions):
    """(d*, n_ends, first_end) of P over S[lo:hi] (the whole sequence or one record; ends relative to lo, None when
    substitutions only finds no window), where S holds BACKGROUND bytes outside `regions` [(x, y), ...] (those
    outside [lo, hi) are ignored) and read(offset, n) reads S back.  Each region's ends (x, y + 2m] are restated from
    S[x - 2m : y + 2m] (clamped to [lo, hi)); every other end scores m.  The regions' end ranges must not overlap."""
    m = len(P)
    first_valid = m if flags & SUB else 0  # the smallest end with a value
    total = hi - lo + 1 - first_valid
    if total <= 0:
        return None
    best, count, first, covered, restated = m + 1, 0, None, [], 0
    for x, y in sorted(regions):
        if y <= lo or x >= hi:
            continue
        assert lo <= x < y <= hi, "a region across a record edge"
        w, z = max(lo, x - 2 * m), min(hi, y + 2 * m)
        assert not covered or covered[-1][1] <= x - lo, "regions closer than 2m"
        covered.append((x - lo, z - lo))
        vals, ends = column(P, read(w, z - w), flags)
        keep = (ends + w > x) & (ends + w <= z)
        vals, ends = vals[keep], ends[keep] + (w - lo)
        restated += ends.size
        if vals.size == 0:
            continue
        d = int(vals.min())
        at = ends[vals == d]
        if d < best:
            best, count, first = d, int(at.size), int(at[0])
        elif d == best:
            best, count, first = d, count + int(at.size), min(first, int(at[0]))
    background = total - restated
    if background and m <= best:
        c = first_valid  # the first end no region covers
        for a, b in covered:
            if a < c <= b:
                c = b + 1
        if m < best:
            best, count, first = m, background, c
        else:
            count, first = count + background, min(first, c)
    return best, count, first


class Plants(object):
    """Regions written into a handle's buffer, undone by writing back what they covered"""

    def __init__(self, hs):
        self.hs, self.saved = hs, []

    def put(self, x, data):
        self.saved.append((x, self.hs.read(x, len(data))))
        self.hs.write(x, data)
        return x, x + len(data)

    def clear(self):
        for x, old in reversed(self.saved):
            self.hs.write(x, old)
        self.saved = []


def region(rng, m, flags, o=0, seam=512):
    """(P, text, at): a random pattern of m symbols over b"ab" and 2 * seam bytes over the same letters whose planted
    match of P ends at `at` = seam + o -- seam_cases' stretched copy for Levenshtein (o % 3 picks its stretch), P
    with one substitution for substitutions only."""
    P, T = next(seam_cases(rng, m, seam, [o]))
    if flags & SUB:
        T = bytearray(b"b" * (2 * seam))
        T[seam + o - m:seam + o] = copy(P, flags)
    return P, bytes(T), seam + o


def copy(P, flags):
    """P itself (Levenshtein: d* = 0) or P with one substitution (substitutions only: d* = 1), over b"ab" """
    v = bytearray(P)
    if flags & SUB:
        v[len(P) // 2] ^= 3  # 'a' <-> 'b'
    return bytes(v)


def place(plants, n, end, T, at):
    """T written so that its end position `at` lands on the sequence's end position `end` (cut at the buffer's
    edges) -> the region"""
    x = end - at
    lo, hi = max(x, 0), min(x + len(T), n)
    return plants.put(lo, T[lo - x:hi - x])


def device_whole(hs, P, flags):
    d, n_ends, first, st = hs.nearest_distance(P, flags)
    assert st["route"] == ("nearest/substitutions-scan" if flags else "nearest/bit-vector-scan")
    return None if (d, n_ends, first) == (NONE32, 0, NONE64) else (d, n_ends, first)


def test_windowed_restatement(cuda_device):
    """The restatement itself, on texts short enough for nearest / hamming over the whole text and for the device:
    regions at the sequence's first and last bytes, two regions 2m apart, ties, record edges, and no region at all.
    The buffer is filled and planted as the large cases fill it."""
    rng = np.random.default_rng(81)
    n = 300_000
    hs = F.Haystack.alloc(n, device=cuda_device)
    hs.fill_synthetic(BACKGROUND, 5)
    plants = Plants(hs)
    for flags in METRICS:
        for m in (24, 40, 100):
            P, T, at = region(rng, m, flags, m % 3)
            _, decoy, _ = region(rng, m, flags, 1)
            regs = [place(plants, n, 200, T, at),  # cut at the sequence's start
                    place(plants, n, n // 3, T, at),
                    place(plants, n, n // 3 + len(T) + 2 * m, T, at),  # as close to the one before as regions may be
                    place(plants, n, 2 * n // 3, decoy, 512),
                    place(plants, n, n // 2 + 9000, copy(P, flags), m),
                    place(plants, n, n - 300, T, at)]  # cut at the sequence's end
            S = hs.read(0, n)
            want = (hamming if flags else nearest)(P, S)
            assert windowed(hs.read, P, flags, 0, n, regs) == want == device_whole(hs, P, flags), (flags, m)
            assert want[0] == int(bool(flags))
            assert windowed(hs.read, P, flags, 0, n, regs[:3]) != want  # (the other regions count)
            # records: every region inside one, clipped to its record, and an empty record
            off = [0, n // 2, n - 1, n]
            hs.set_records(off)
            dist, end, _ = hs.nearest_per_record(P, flags)
            for r in range(3):
                lo, hi = off[r], off[r + 1] - 1
                got = windowed(hs.read, P, flags, lo, hi, [(max(x, lo), min(y, hi)) for x, y in regs if x < hi < y or
                                                           lo <= x < hi])
                if r == 2:
                    assert got == (None if flags else (m, 1, 0))
                else:
                    assert got == (hamming if flags else nearest)(P, S[lo:hi]), (flags, m, r)
                assert (int(dist[r]), int(end[r])) == ((-1, -1) if got is None else (got[0], got[2])), (flags, m, r)
            hs.set_records(None)
            plants.clear()
            closed = (m, n - m + 1, m) if flags else (m, n + 1, 0)
            assert windowed(hs.read, P, flags, 0, n, []) == closed == device_whole(hs, P, flags)
            # regions of a letter P lacks, at the sequence's start and one byte long: their best ties with the
            # background's m (substitutions only: the region holds the first end)
            regs = [plants.put(0, b"c" * 3), plants.put(n // 2, b"c")]
            whole = (hamming if flags else nearest)(P, hs.read(0, n))
            assert windowed(hs.read, P, flags, 0, n, regs) == closed == whole
            assert device_whole(hs, P, flags) == closed
            plants.clear()
    hs.close()


def test_past_2_32_whole_sequence(cuda_device):
    """Best ends at 2^32 - 1, 2^32 and 2^32 + 1, across a segment, a tile and a grid-pass seam above 2^32 and at the
    sequence's last byte, each as a copy of the pattern and as a stretched copy, alone and tied with one below 2^32;
    then the batch over the same sequence -- both word classes and the single scan of a 100-symbol pattern -- with the
    best ends at its warp-segment seams and ties between patterns."""
    needs_real_gpu("a 4.4 GB sequence")
    rng = np.random.default_rng(82)
    sms = sm_count()
    n = big_n(sms)
    assert seg_of(n, sms) == MAX_SEG
    seg, tile = MAX_SEG, THREADS * MAX_SEG
    hs = F.Haystack.alloc(n, device=cuda_device)
    hs.fill_synthetic(BACKGROUND, 6)
    plants = Plants(hs)
    low = G31 + 12345  # where a copy below 2^32 ties
    for flags in METRICS:
        for m in (24, 40, 100):
            grid_pass = grid_of(n, m, sms) * tile
            passes = (n - (1 << 19)) // grid_pass * grid_pass
            assert passes > G32
            seams = [(G32 // seg + 3) * seg, (G32 // tile + 2) * tile, passes]
            for end in [G32 - 1, G32, G32 + 1, n] + [s + o for s in seams for o in (0, 1, m)]:
                P, T, at = region(rng, m, flags, end % 3)
                for kind, (text, t_at) in (("copy", (copy(P, flags), m)), ("stretched", (T, at))):
                    for tie in (False, True):
                        regs = [place(plants, n, end, text, t_at)]
                        if tie:
                            regs.append(place(plants, n, low, text, t_at))
                        want = windowed(hs.read, P, flags, 0, n, regs)
                        if kind == "copy":
                            assert want == (int(bool(flags)), 1 + tie, low if tie else end), (flags, m, end, want)
                        assert device_whole(hs, P, flags) == want, (flags, m, end, kind, tie)
                        plants.clear()
    # the batch: 20 / 24 / 24 / 32 symbols (one group; patterns 1 and 5 equal: a tie between patterns), 40 / 64
    # symbols (one group of the 64-bit class), 100 symbols (the single scan); copies end at warp-segment seams past
    # 2^32, pattern 0 ties with a copy below 2^32, and the only copy of pattern 6 ends at the last byte
    s32, s64 = warp_seg(n, 1, False, sms), warp_seg(n, 1, True, sms)
    for flags in METRICS:
        pats = [rand(rng, b"ab", m) for m in (20, 24, 40, 64, 100)]
        pats += [pats[1], rand(rng, b"ab", 32)]
        ends = [(G32 // s32 + 1) * s32, (G32 // s32 + 2) * s32 + 1, (G32 // s64 + 1) * s64,
                (G32 // s64 + 2) * s64 + 40, (G32 // seg + 1) * seg]
        regs = [place(plants, n, e, copy(P, flags), len(P)) for e, P in zip(ends, pats)]
        regs.append(place(plants, n, low, copy(pats[0], flags), 20))
        regs.append(place(plants, n, n, copy(pats[6], flags), 32))
        dist, end, st = hs.nearest_distance_batch(pats, flags)
        want = [windowed(hs.read, P, flags, 0, n, regs) for P in pats]
        assert [w[0] for w in want] == [int(bool(flags))] * 7
        assert [w[2] for w in want] == [low] + ends[1:] + [ends[1], n]
        assert dist.tolist() == [w[0] for w in want] and end.tolist() == [w[2] for w in want], (flags, want)
        assert st["bytes_scanned"] == 3 * n
        plants.clear()
    hs.close()


def test_n_ends_past_2_32(cuda_device):
    """No plant and a pattern absent from the sequence: every end is at m."""
    needs_real_gpu("a 4.4 GB sequence")
    rng = np.random.default_rng(83)
    n = big_n(sm_count())
    hs = F.Haystack.alloc(n, device=cuda_device)
    hs.fill_synthetic(BACKGROUND, 7)
    for m in (24, 40, 100):
        P = rand(rng, b"ACGT", m)
        assert device_whole(hs, P, 0) == (m, n + 1, 0) == windowed(hs.read, P, 0, 0, n, [])
        assert device_whole(hs, P, SUB) == (m, n - m + 1, m) == windowed(hs.read, P, SUB, 0, n, [])
    hs.close()


def test_intermediate_segment_lengths(cuda_device):
    """Two sequence lengths for which the host picks a segment between the shortest and the longest: the planted match
    ends at every offset -2m .. 2m from a segment seam and from a tile seam, as a stretched copy (Levenshtein) and as a
    copy whose end is the unique best (both metrics)."""
    needs_real_gpu("140 MB and 370 MB sequences")
    rng = np.random.default_rng(84)
    sms = sm_count()
    for seg in (1040, 2720):
        n = (seg - 8) * sms * 1024 + 5
        assert seg_of(n, sms) == seg
        hs = F.Haystack.alloc(n, device=cuda_device)
        hs.fill_synthetic(BACKGROUND, 8)
        plants = Plants(hs)
        for flags in METRICS:
            for m in (24, 40):
                for seam in (7 * seg, 3 * THREADS * seg):
                    for o in range(-2 * m, 2 * m + 1):
                        P, T, at = region(rng, m, flags, o)
                        kinds = [("copy", copy(P, flags), m)] + ([] if flags else [("stretched", T, at)])
                        for kind, text, t_at in kinds:
                            regs = [place(plants, n, seam + o, text, t_at)]
                            want = windowed(hs.read, P, flags, 0, n, regs)
                            if kind == "copy":
                                assert want == (int(bool(flags)), 1, seam + o), (seg, flags, m, seam, o, want)
                            else:
                                assert abs(want[2] - (seam + o)) <= 2 * m, (seg, m, seam, o, want)
                            assert device_whole(hs, P, flags) == want, (seg, flags, m, seam, o, kind)
                            plants.clear()
        hs.close()


def restated_rows(hs, pats, flags, off, regs):
    """(D, E): windowed's (d*, first_end) of every pattern over every record of the set `off`, -1 without a value"""
    D = np.full((len(pats), len(off) - 1), -1, np.int64)
    E = D.copy()
    for i, P in enumerate(pats):
        for r in range(len(off) - 1):
            got = windowed(hs.read, P, flags, off[r], off[r + 1] - 1, regs)
            if got is not None:
                D[i, r], E[i, r] = got[0], got[2]
    return D, E


def check_cols(cols, want, ctx=()):
    for name, got, exp in zip(("pattern", "dist", "end", "second_pattern", "second_dist"), cols, want):
        bad = np.flatnonzero(np.asarray(got) != np.asarray(exp))
        assert bad.size == 0, ctx + (name, bad[:5], np.asarray(got)[bad[:5]], np.asarray(exp)[bad[:5]])


def test_record_of_2_32_minus_1_bytes(cuda_device):
    """Record 0 is [0, 2^32 - 1): its best end is its last byte (2^32 - 1), a second region ends at 2^31, and a
    100-symbol pattern (the fold) wins there by index over its own 24-symbol suffix; short records follow, one of them
    empty.  A record of 2^32 bytes is refused, and the handle then answers as before."""
    needs_real_gpu("a 4.3 GB record")
    rng = np.random.default_rng(85)
    P100 = rand(rng, b"ACGT", 100)
    P40, P20 = rand(rng, b"ACGT", 40), rand(rng, b"ACGT", 20)
    pats = [P40, P100, P100[-24:], P20]
    v24 = P100[-24:-1] + (b"A" if P100[-1:] != b"A" else b"C")
    short = [b"", rand(rng, b"ACGT", 130) + P20, b"A", rand(rng, b"ACGT", 200) + v24 + b"ACGT" * 9]
    off = [0, G32]
    for r in short:
        off.append(off[-1] + len(r) + 1)
    n = off[-1]
    hs = F.Haystack.alloc(n, device=cuda_device)
    hs.fill_synthetic(BACKGROUND, 9)
    for o in off[1:]:
        hs.write(o - 1, b"\0")
    regs = [(o, o + len(r)) for o, r in zip(off[1:], short) if r]
    for o, r in zip(off[1:], short):
        hs.write(o, r)
    regs.append((G32 - 1 - 100, G32 - 1))
    hs.write(G32 - 1 - 100, P100)
    v40 = P40[:20] + (b"A" if P40[20:21] != b"A" else b"C") + P40[21:]
    regs.append((G31 - 40, G31))
    hs.write(G31 - 40, v40)
    before = {}
    for flags in METRICS:
        hs.set_records(off)
        D, E = restated_rows(hs, pats, flags, off, regs)
        assert D[:3, 0].tolist() == [1, 0, 0] and E[1:3, 0].tolist() == [G32 - 1, G32 - 1]
        assert E[0, 0] == G31
        for i, P in enumerate(pats):
            dist, end, _ = hs.nearest_per_record(P, flags)
            assert dist.tolist() == D[i].tolist() and end.tolist() == E[i].tolist(), (flags, i)
            before[flags, i] = dist.tolist(), end.tolist()
        cols, st = hs.nearest_best_per_record(pats, flags)
        want = (ham_reduce_rows if flags else lev_reduce_rows)(D, E)
        check_cols(cols, want, (flags,))
        assert [int(c[0]) for c in cols] == [1, 0, G32 - 1, 2, 0]  # the fold wins by index over its suffix
        before[flags] = [c.tolist() for c in cols]
        # record 0 of 2^32 bytes: both calls refuse, and the handle keeps its answers
        hs.set_records([0, G32 + 1] + off[3:])
        with pytest.raises(F.UnsupportedError):
            hs.nearest_per_record(P40, flags)
        with pytest.raises(F.UnsupportedError):
            hs.nearest_best_per_record(pats, flags)
        hs.set_records(off)
        assert [c.tolist() for c in hs.nearest_best_per_record(pats, flags)[0]] == before[flags]
        dist, end, _ = hs.nearest_per_record(P40, flags)
        assert (dist.tolist(), end.tolist()) == before[flags, 0]
    hs.close()


def oracle_columns(hs, pats, lim4, off, windows):
    """The six columns of fzb_best_per_record restated by reduce_lists over the oracle's lists in `windows`
    [(record, lo, hi), ...] read back from the handle; the records' other bytes are BACKGROUND, where no pattern
    matches."""
    s, i, d, l = lim4
    lists = [{} for _ in pats]
    for r, lo, hi in windows:
        text = hs.read(lo, hi - lo)
        for q, P in enumerate(pats):
            ms = oracle.find_near_matches(P, text, max_substitutions=s, max_insertions=i, max_deletions=d,
                                          max_l_dist=l)
            shift = lo - off[r]
            lists[q].setdefault(r, []).extend((a + shift, b + shift, dd) for a, b, dd in ms)
    lists = [{r: ms for r, ms in d.items() if ms} for d in lists]
    return reduce_lists(lists, len(off) - 1)


def test_record_of_2_31_minus_1_bytes_best_per_record(cuda_device):
    """fzb_best_per_record over a record of 2^31 - 1 bytes: the best match ends at its last byte, so its start is
    2^31 - 1 - m in the 31-bit field; a different pattern is the runner-up, with a start above 2^30.  A record of
    2^31 bytes is refused, and the handle then answers as before."""
    needs_real_gpu("a 2.1 GB record")
    rng = np.random.default_rng(86)
    P, Q, R = rand(rng, b"ACGT", 24), rand(rng, b"ACGT", 20), rand(rng, b"ACGT", 30)
    pats = [Q, P, R]
    short = [rand(rng, b"ACGT", 150) + R, b"", rand(rng, b"ACGT", 90)]
    off = [0, G31]
    for r in short:
        off.append(off[-1] + len(r) + 1)
    n = off[-1]
    hs = F.Haystack.alloc(n, device=cuda_device)
    hs.fill_synthetic(BACKGROUND, 10)
    for o in off[1:]:
        hs.write(o - 1, b"\0")
    for o, r in zip(off[1:], short):
        hs.write(o, r)
    vq = Q[:10] + (b"A" if Q[10:11] != b"A" else b"G") + Q[11:]
    q_end = (1 << 30) + 777_777
    hs.write(q_end - 20, vq)
    hs.write(G31 - 1 - 24, P)
    hs.set_records(off)
    windows = [(0, q_end - 80, q_end + 60), (0, G31 - 200, G31 - 1)] + \
        [(r + 1, off[r + 1], off[r + 2] - 1) for r in range(len(short))]
    for lim4 in ((2, 2, 2, 2), (2, 0, 0, 2)):
        want = oracle_columns(hs, pats, lim4, off, windows)
        assert [want[k][0] for k in NAMES] == [1, G31 - 1 - 24, G31 - 1, 0, 0, 1], lim4
        got, _ = hs.best_per_record(pats, *[[x] * 3 for x in lim4])
        for name, col in zip(NAMES, got):
            assert col.tolist() == want[name], (lim4, name)
        hs.set_records([0, G31 + 1] + off[3:])  # record 0 of 2^31 bytes
        with pytest.raises(F.UnsupportedError):
            hs.best_per_record(pats, *[[x] * 3 for x in lim4])
        hs.set_records(off)
        again, _ = hs.best_per_record(pats, *[[x] * 3 for x in lim4])
        assert all(a.tolist() == b.tolist() for a, b in zip(again, got)), lim4
    hs.close()


MAX_PATTERNS = 65535


def many_patterns(rng, small):
    """65 535 patterns of 20-64 symbols over bytes 128-255, absent from every text (the dead ones), but for the live
    ones over ACGT: ordinals 0, 31-33, 32 767-32 769, 65 500-65 534, the first and last lanes of some groups in the
    host's (class, length) order, and random others.  Ordinal 65 534 has 100 symbols (the fold path), ordinal 65 533
    is its 30-symbol suffix with one substitution at the front."""
    ms = rng.integers(20, 65, size=MAX_PATTERNS)
    ms[-2:] = (30, 100)
    c32 = sorted((i for i in range(MAX_PATTERNS) if ms[i] <= 32), key=lambda i: ms[i])
    c64 = sorted((i for i in range(MAX_PATTERNS) if 32 < ms[i] <= 64), key=lambda i: ms[i])
    lanes = c32 + [None] * (-len(c32) % 32) + c64
    live = {0, 31, 32, 33, 32767, 32768, 32769} | set(range(65500 if not small else 65525, MAX_PATTERNS))
    live |= {lanes[32 * g + k] for g in (0, 1, 100, len(c32) // 32, len(c32) // 32 + 1, len(lanes) // 32 - 1)
             for k in (0, 31) if 32 * g + k < len(lanes) and lanes[32 * g + k] is not None}
    live |= set(rng.integers(0, MAX_PATTERNS, size=200 if not small else 20).tolist())
    dead = np.arange(128, 256, dtype=np.uint8)
    pats = [rand(rng, b"ACGT", int(m)) if i in live else bytes(dead[rng.integers(0, 128, size=int(m))])
            for i, m in enumerate(ms)]
    pats[-2] = (b"A" if pats[-1][70:71] != b"A" else b"C") + pats[-1][71:]
    return pats, sorted(live)


def closed_form(pats, live, lens, flags):
    """(D, E) of every pattern over texts of the given lengths: the dead patterns' in closed form (Levenshtein: m at
    the end position 0; substitutions only: m at the first window, none in a text shorter than m), the live rows -1"""
    ms = np.array([len(P) for P in pats], np.int64)[:, None]
    lens = np.asarray(lens, np.int64)[None, :]
    if flags & SUB:
        fits = lens >= ms
        D, E = np.where(fits, ms, -1), np.where(fits, ms, -1)
    else:
        D, E = np.broadcast_to(ms, (len(pats), lens.size)).copy(), np.zeros((len(pats), lens.size), np.int64)
    D[live], E[live] = -1, -1
    return D, E


def stacked(P, recs, flags):
    """(dist, first_end) of P in every record, -1 without a value: one restatement over the records padded with 'x'"""
    L = max([len(r) for r in recs] + [1])
    rows = np.full((len(recs), L), ord("x"), np.uint8)
    for i, r in enumerate(recs):
        rows[i, :len(r)] = np.frombuffer(r, np.uint8)
    lens = np.array([len(r) for r in recs])[:, None]
    vals, ends = column(P, rows, flags)
    if ends.size == 0:
        return np.full(len(recs), -1), np.full(len(recs), -1)
    vals = np.where(ends[None, :] <= lens, vals, 1 << 20)  # (substitutions only: windows past the record's end)
    at = vals.argmin(axis=1)
    d = vals[np.arange(len(recs)), at]
    return np.where(d < 1 << 20, d, -1), np.where(d < 1 << 20, ends[at], -1)


def test_65535_patterns(cuda_device, small=False):
    """65 535 patterns, the largest batch, over a short sequence and over a short record set; records where the
    winner and runner-up are ordinals 65 533 and 65 534 either way round, tied at 0 and broken by ordinal, the fold
    pattern at ordinal 65 534; 65 536 patterns refused."""
    rng = np.random.default_rng(87)
    pats, live = many_patterns(rng, small)
    top, suffix = pats[-1], pats[-2]
    recs = [rand(rng, b"ACGT", int(k)) for k in rng.integers(0, 120 if small else 300, size=12 if small else 100)]
    special = [i for i in (0, 31, 32, 33, 32767, 32768, 32769, 65500, 65525, 65532) if i in set(live)]
    planted = special + [i for i in rng.permutation(live).tolist() if i not in special]
    for k, i in enumerate(planted[:len(recs) // 2]):  # live patterns planted whole or with one substitution
        P = bytearray(pats[i])
        if k % 2:
            P[len(P) // 2] = ord("T") if P[len(P) // 2] != ord("T") else ord("G")
        recs[2 * k] = recs[2 * k][:40] + bytes(P) + recs[2 * k][40:]
    recs += [b"w" * 30 + top + b"w" * 30,                  # 65 534 exact (the fold), 65 533 one substitution
             b"w" * 30 + top + b"w" + suffix + b"w",      # both exact: the tie goes to 65 533
             b"", b"A", suffix]
    S = b"".join(recs[::-1])
    hs = F.Haystack.alloc(len(joined(recs)[0]), device=cuda_device)
    for flags in METRICS:
        hs.set_records(None)
        hs.upload(S)
        dist, end, st = hs.nearest_distance_batch(pats, flags)
        D, E = closed_form(pats, live, [len(S)], flags)
        for i in live:
            got = (hamming if flags else nearest)(pats[i], S)
            D[i, 0], E[i, 0] = got[0], got[2]
        assert dist.tolist() == D[:, 0].tolist() and end.tolist() == E[:, 0].tolist(), flags
        buf, off = joined(recs)
        hs.upload(buf)
        hs.set_records(off)
        cols, st = hs.nearest_best_per_record(pats, flags)
        D, E = closed_form(pats, live, [len(r) for r in recs], flags)
        for i in live:
            D[i], E[i] = stacked(pats[i], recs, flags)
        want = (ham_reduce_rows if flags else lev_reduce_rows)(D, E)
        check_cols(cols, want, (flags,))
        R = len(recs)
        assert [int(c[R - 5]) for c in want] == [65534, 0, 130, 65533, 1]
        assert [int(c[R - 4]) for c in want] == [65533, 0, 161, 65534, 0]
        with pytest.raises(F.UnsupportedError):
            hs.nearest_best_per_record(pats + [b"A"], flags)
        hs.set_records(None)
        with pytest.raises(F.UnsupportedError):
            hs.nearest_distance_batch(pats + [b"A"], flags)
    hs.close()
