"""find_near_matches_batch with per-pattern limits, against a stand-in haystack that answers the C-ABI from the CPU
oracle (fake_backend) and adds the substitutions-only batch: the dispatch by search class, the limit each class
receives, input order, errors and the fallback for wide alphabets, on a box without a GPU."""
import pytest

import oracle
from fake_backend import FakeHaystack, FakePinnedBuffer
from fuzzysearch_b200 import _native as F, find_near_matches, find_near_matches_batch

CALLS = []


class HamBatchHaystack(FakeHaystack):
    """FakeHaystack plus fzb_search_hamming_batch (the oracle, per pattern); records the calls it answers."""

    def search_hamming_batch(self, pats, ks, flags=0):
        CALLS.append(("hamming_batch", [F.as_u8(p).tobytes() for p in pats], [int(k) for k in ks]))
        return [self.search_hamming(p, int(k)) for p, k in zip(pats, ks)], {}

    def search_levenshtein_batch(self, pats, ks, flags=0):
        CALLS.append(("levenshtein_batch", [F.as_u8(p).tobytes() for p in pats], [int(k) for k in ks]))
        return super().search_levenshtein_batch(pats, ks, flags)

    def search_generic(self, p, subs, ins, dels, l, flags=0):
        CALLS.append(("generic", F.as_u8(p).tobytes(), (subs, ins, dels, l)))
        return super().search_generic(p, subs, ins, dels, l, flags)


@pytest.fixture()
def ham_batch_device(monkeypatch):
    from fuzzysearch_b200 import search
    monkeypatch.setattr(F, "Haystack", HamBatchHaystack)
    monkeypatch.setattr(F, "PinnedBuffer", FakePinnedBuffer)
    monkeypatch.setattr(F, "device_count", lambda: 1)
    saved = dict(search._WORKSPACE)
    search._WORKSPACE.clear()
    del CALLS[:]
    yield
    search._WORKSPACE.clear()
    search._WORKSPACE.update(saved)


SEQ = b"xxGATTACAxxGATTTCAxxGATACAxxCATTACAGxxGATTACA" * 3
PATS = [b"GATTACA", b"GATTACA", b"CATTACAG", b"GATTTCA", b"ATTAC"]
LIMITS = [dict(max_l_dist=0),
          dict(max_substitutions=1, max_insertions=0, max_deletions=0),
          dict(max_l_dist=1),
          dict(max_substitutions=1, max_insertions=1, max_deletions=0, max_l_dist=1),
          dict(max_substitutions=2, max_insertions=0, max_deletions=0, max_l_dist=1)]


def per_pattern(limits):
    return {key: [d.get(key) for d in limits]
            for key in ("max_substitutions", "max_insertions", "max_deletions", "max_l_dist")}


def test_each_class_takes_its_own_path(ham_batch_device):
    got = find_near_matches_batch(PATS, SEQ, **per_pattern(LIMITS))
    assert got == [find_near_matches(p, SEQ, **d) for p, d in zip(PATS, LIMITS)]
    assert got[1] and got[4] and got[0]
    calls = [c for c in CALLS if c[0] != "generic" or c[1] == PATS[3]][:3]
    # exact and Levenshtein share one batch, with the normalised max_l_dist; substitutions-only ones another, with
    # min(max_l_dist, max_substitutions); the generic one runs on its own
    assert calls[0] == ("levenshtein_batch", [PATS[0], PATS[2]], [0, 1])
    assert calls[1] == ("hamming_batch", [PATS[1], PATS[4]], [1, 1])
    assert calls[2] == ("generic", PATS[3], (1, 1, 0, 1))


def test_max_l_dist_only_takes_the_levenshtein_batch(ham_batch_device):
    got = find_near_matches_batch(PATS, SEQ, [0, 1, 2, 1, 0])
    assert got == [find_near_matches(p, SEQ, max_l_dist=k) for p, k in zip(PATS, [0, 1, 2, 1, 0])]
    assert [c[0] for c in CALLS] == ["levenshtein_batch"]
    assert find_near_matches_batch(PATS, SEQ, 1) == [find_near_matches(p, SEQ, max_l_dist=1) for p in PATS]


def test_substitutions_only_batch_results_in_input_order(ham_batch_device):
    ks = [0, 1, 2, 1, 3]
    got = find_near_matches_batch(PATS, SEQ, max_substitutions=ks, max_insertions=0, max_deletions=0)
    for p, k, ms in zip(PATS, ks, got):
        want = oracle.find_near_matches(p, SEQ, k, 0, 0, None)
        assert [(m.start, m.end, m.dist) for m in ms] == want
        assert all(m.matched == SEQ[m.start:m.end] for m in ms)
    assert [c[0] for c in CALLS] == ["levenshtein_batch", "hamming_batch"]  # (k = 0: ExactSearch)
    assert CALLS[1][2] == [1, 2, 1, 3]


@pytest.mark.parametrize("bad", [dict(max_substitutions=-1, max_insertions=0, max_deletions=0),
                                 dict(max_substitutions=2), dict(max_substitutions=1, max_deletions=0), dict(),
                                 dict(max_l_dist=1.5), dict(max_substitutions=[1, None, 1, 1, 1], max_insertions=0,
                                                            max_deletions=0)])
def test_invalid_limits_raise_like_find_near_matches(ham_batch_device, bad):
    with pytest.raises(Exception) as batch:
        find_near_matches_batch(PATS, SEQ, **bad)
    single = {k: (v[1] if isinstance(v, list) else v) for k, v in bad.items()}
    with pytest.raises(Exception) as one:
        find_near_matches(PATS[1], SEQ, **single)
    assert type(batch.value) is type(one.value) and str(batch.value) == str(one.value)
    assert not CALLS


def test_length_mismatch_and_empty_patterns(ham_batch_device):
    with pytest.raises(ValueError, match="one max_substitutions per subsequence"):
        find_near_matches_batch(PATS, SEQ, max_substitutions=[1, 2], max_insertions=0, max_deletions=0)
    with pytest.raises(ValueError, match="Given subsequence is empty!"):
        find_near_matches_batch([b"ACGT", b""], SEQ, max_substitutions=1, max_insertions=0, max_deletions=0)
    with pytest.raises(ValueError, match="subsequence must not be empty"):
        find_near_matches_batch([b"ACGT", b""], SEQ, max_l_dist=0)
    assert find_near_matches_batch([], SEQ, max_substitutions=1, max_insertions=0, max_deletions=0) == []


def test_wide_alphabet_fallback_covers_every_class(ham_batch_device):
    """More than 255 distinct symbols over the patterns: each pattern goes through find_near_matches on its own."""
    pats = ["".join(chr(0x1000 + 40 * j + i) for i in range(40)) for j in range(8)]
    seq = "".join(pats) * 2
    limits = [LIMITS[j % len(LIMITS)] for j in range(len(pats))]
    got = find_near_matches_batch(pats, seq, **per_pattern(limits))
    assert got == [find_near_matches(p, seq, **d) for p, d in zip(pats, limits)]
    assert all(len(g) == 2 for g in got)
    assert "hamming_batch" not in [c[0] for c in CALLS]
