"""The Python layers above the C-ABI where they take a path of their own: the pattern-by-pattern fallbacks of
align_in_each and nearest_pattern_in_each when the patterns have no common byte alphabet (more than 255 distinct
wide symbols over them), the row checks of align_in_each, and the pattern packing of the Haystack batch calls at
their empty edges.  Each fallback row is compared with the same call on that read (or pattern) alone, which takes
the ordinary one-alphabet path.  Replayed on the emulator by tests/test_emu_python_layers.py."""
import numpy as np
import pytest

from fuzzysearch_b200 import (DeviceSequenceSet, _native as F, align_in_each, align_matches, best_match_in_each,
                              nearest_distance_in_each, nearest_pattern_in_each)
from test_gpu_records import joined

pytestmark = pytest.mark.gpu

SYMBOLS = [chr(0x400 + i) for i in range(260)]


def wide_case(rng, n_reads, at=None):
    """52 patterns of 5 symbols each, 260 distinct symbols over all of them, and reads over the same symbols, each
    holding one pattern with one substitution (`at`: 'start' / 'end' puts it there, None anywhere), plus an empty
    read and one shorter than every pattern."""
    pats = ["".join(SYMBOLS[5 * i:5 * i + 5]) for i in range(52)]
    reads = []
    for r in range(n_reads):
        p = list(pats[(7 * r) % 52])
        p[int(rng.integers(0, 5))] = SYMBOLS[int(rng.integers(0, 260))]
        head = "".join(SYMBOLS[int(x)] for x in rng.integers(0, 260, size=int(rng.integers(0, 12))))
        tail = "".join(SYMBOLS[int(x)] for x in rng.integers(0, 260, size=int(rng.integers(0, 12))))
        reads.append("".join(p) + tail if at == "start" else head + "".join(p) if at == "end" else
                     head + "".join(p) + tail)
    return pats, reads + ["", SYMBOLS[3] + SYMBOLS[9]]


def columns(al, r):
    return (int(al.start[r]), int(al.end[r]), int(al.dist[r]), int(al.substitutions[r]), int(al.insertions[r]),
            int(al.deletions[r]), al.cigar[r])


def test_align_in_each_without_a_common_alphabet(cuda_device, small=False):
    """align_in_each over BestMatches and NearestPatterns rows of 260-symbol pattern sets: every row is what
    align_matches / align_in_each give on that read alone."""
    rng = np.random.default_rng(31)
    pats, reads = wide_case(rng, 30 if small else 120)
    best = best_match_in_each(pats, reads, 1)
    assert (best.pattern[:-2] >= 0).all()
    al = align_in_each(pats, reads, best, 1)
    for r in range(len(reads)):
        if best.pattern[r] < 0:
            assert al[r] is None and al.cigar[r] == ""
            continue
        p, m = best[r]
        assert align_matches(pats[p], reads[r], [m], max_l_dist=1) == [al.cigar[r]], r
        assert (int(al.start[r]), int(al.end[r])) == (m.start, m.end), r
        assert al.substitutions[r] + al.insertions[r] + al.deletions[r] == al.dist[r] <= m.dist
    for subs in (False, True):
        near = nearest_pattern_in_each(pats, reads, substitutions_only=subs)
        resident = DeviceSequenceSet(reads)
        al = align_in_each(pats, resident, near, substitutions_only=subs)
        resident.close()
        for r in range(len(reads)):
            p = int(near.pattern[r])
            if p < 0:
                assert subs and al[r] is None, r
                continue
            one = nearest_distance_in_each(pats[p], [reads[r]], substitutions_only=subs)
            assert (int(one.dist[0]), int(one.end[0])) == (int(near.dist[r]), int(near.end[r])), (subs, r)
            alone = align_in_each(pats[p], [reads[r]], one, substitutions_only=subs)
            assert columns(al, r) == columns(alone, 0), (subs, r)


def reduce_anchored(loop, n):
    """The winner (the smallest distance, then the smallest index) and the runner-up among the other patterns of
    every read, from per-pattern NearestDistances; the winner's start and end with it; patterns without a distance
    (-1) left out -> (pattern, dist, start, end, second_pattern, second_dist) lists."""
    out = [[] for _ in range(6)]
    for r in range(n):
        ranked = sorted((int(x.dist[r]), i) for i, x in enumerate(loop) if x.dist[r] >= 0)
        (d, i), (d2, i2) = (ranked + [(-1, -1)] * 2)[:2]
        row = (i, d, int(loop[i].start[r]) if i >= 0 else -1, int(loop[i].end[r]) if i >= 0 else -1, i2, d2)
        for c, v in zip(out, row):
            c.append(v)
    return out


@pytest.mark.parametrize("anchor", ["start", "end"])
def test_anchored_nearest_patterns_without_a_common_alphabet(cuda_device, anchor, small=False):
    """nearest_pattern_in_each(..., anchor=) over 260 distinct symbols equals the reduction of
    nearest_distance_in_each(p, reads, anchor=) over the patterns, the winner's start and end included; its rows
    align as align_in_each aligns them on that read alone."""
    rng = np.random.default_rng(32 if anchor == "start" else 33)
    pats, reads = wide_case(rng, 24 if small else 80, at=anchor)
    resident = DeviceSequenceSet(reads)
    for subs in (False, True):
        rows = nearest_pattern_in_each(pats, reads, substitutions_only=subs, anchor=anchor)
        loop = [nearest_distance_in_each(p, resident, substitutions_only=subs, anchor=anchor) for p in pats]
        want = reduce_anchored(loop, len(reads))
        got = [c.tolist() for c in (rows.pattern, rows.dist, rows.start, rows.end, rows.second_pattern,
                                    rows.second_dist)]
        assert got == want, (anchor, subs)
        al = align_in_each(pats, resident, rows, substitutions_only=subs)
        for r in range(len(reads)):
            p = int(rows.pattern[r])
            if p < 0:
                assert al[r] is None
                continue
            assert (int(al.start[r]), int(al.end[r]), int(al.dist[r])) == \
                (int(rows.start[r]), int(rows.end[r]), int(rows.dist[r])), (anchor, subs, r)
            if r < 8:
                one = nearest_distance_in_each(pats[p], [reads[r]], substitutions_only=subs, anchor=anchor)
                alone = align_in_each(pats[p], [reads[r]], one, substitutions_only=subs)
                assert columns(al, r) == columns(alone, 0), (anchor, subs, r)
    resident.close()


def test_align_in_each_row_checks(cuda_device):
    """Rows of the wrong length and rows naming an unknown pattern are refused with the same ValueError, on a list
    and on a resident set; a `sequences` of the wrong type is refused first."""
    pats = [b"GATTACA", b"TTGACCA", b"ACGTACG"]
    reads = [b"xxGATTACAxx", b"TTGACCAyy", b"", b"ACGTACG"]
    near = nearest_pattern_in_each(pats, reads)
    best = best_match_in_each(pats, reads, 1)
    resident = DeviceSequenceSet(reads)
    for seqs in (reads, resident):
        with pytest.raises(ValueError, match="^one row per sequence expected$"):
            align_in_each(pats, seqs, nearest_pattern_in_each(pats, reads[:3]))
        with pytest.raises(ValueError, match="^one row per sequence expected$"):
            align_in_each(pats, seqs, best_match_in_each(pats, reads + [b"GATTACA"], 1), 1)
        with pytest.raises(ValueError, match="^a row names pattern 2 of 2$"):
            align_in_each(pats[:2], seqs, near)
        with pytest.raises(ValueError, match="^a row names pattern 2 of 2$"):
            align_in_each(pats[:2], seqs, best, 1)
        assert align_in_each(pats, seqs, near).cigar == align_in_each(pats, reads, near).cigar
    resident.close()
    for seqs in ("xxxx", b"xxxx", 4, None):
        with pytest.raises(TypeError, match="^sequences must be a list, a tuple or a DeviceSequenceSet$"):
            align_in_each(pats, seqs, near)
        with pytest.raises(TypeError, match="^sequences must be a list, a tuple or a DeviceSequenceSet$"):
            align_in_each(pats[:2], seqs, nearest_pattern_in_each(pats, reads[:3]))
    with pytest.raises(TypeError, match="^rows must be"):
        align_in_each(pats, "xxx", [1, 2, 3])


def test_pattern_packing_at_its_empty_edges(cuda_device):
    """The Haystack calls that pack a list of patterns: no patterns at all is answered, a list of empty patterns is
    refused as a NULL pattern blob, and the handle then answers a search as before."""
    recs = [b"xxGATTACAxx", b"TTGACCA", b""]
    buf, off = joined(recs)
    hs = F.Haystack.from_host(buf)
    hs.set_records(off)
    lev = [1 << 29] * 4
    rec = F.F_PER_RECORD
    assert hs.search_levenshtein_batch([], [], rec)[0] == []
    assert hs.search_hamming_batch([], [], rec)[0] == []
    assert hs.search_generic_batch([], [], [], [], [], rec)[0] == []
    cols, st = hs.best_per_record([], [], [], [], [])
    assert [c.tolist() for c in cols] == [[-1] * 3] * 6 and st["route"] == "batch"
    plain = F.Haystack.from_host(buf)  # (fzb_nearest_distance_batch takes no record set)
    dist, end, _ = plain.nearest_distance_batch([])
    assert dist.size == end.size == 0
    cols, _ = hs.nearest_best_per_record([])
    assert [c.tolist() for c in cols] == [[-1] * 3] * 5
    cols, ops, oo, _ = hs.align([], [], [], [], [], [], [], [], [])
    assert [c.size for c in cols] == [0] * 5 and oo.tolist() == [0]
    for call in (lambda: hs.search_levenshtein_batch([b""], [1], rec),
                 lambda: hs.search_hamming_batch([b""], [1], rec),
                 lambda: hs.search_generic_batch([b""], [1], [1], [1], [1], rec),
                 lambda: hs.best_per_record([b""], *[[x] for x in lev]),
                 lambda: plain.nearest_distance_batch([b""]),
                 lambda: hs.nearest_best_per_record([b""]),
                 lambda: hs.align([b""], *[[x] for x in lev], [], [], [], [])):
        with pytest.raises(ValueError, match="^NULL argument$"):
            call()
    rs, st = hs.search_levenshtein_batch([b"GATTACA"], [1], rec)
    assert rs[0].triples()[0][:2] == (2, 9) and st["route"] == "batch"
    for r in rs:
        r.close()
    hs.close()
    plain.close()
