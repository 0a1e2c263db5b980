"""find_near_matches_batch's dispatch of generic-limit patterns, against a stand-in haystack that answers the C-ABI
from the CPU oracle (fake_backend) and adds the three batch calls: generic patterns reach search_generic_batch with
their normalised limits, in input order, on a box without a GPU."""
import pytest

from fake_backend import FakeHaystack, FakePinnedBuffer
from fuzzysearch_b200 import _native as F, find_near_matches, find_near_matches_batch

CALLS = []


class GenericBatchHaystack(FakeHaystack):
    """FakeHaystack plus the Hamming and generic batches (the oracle, per pattern); records the calls it answers."""

    def search_generic_batch(self, pats, subs, ins, dels, l, flags=0):
        lims = [tuple(int(x) for x in t) for t in zip(subs, ins, dels, l)]
        CALLS.append(("generic_batch", [F.as_u8(p).tobytes() for p in pats], lims))
        return [FakeHaystack.search_generic(self, p, *lim) for p, lim in zip(pats, lims)], {}

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
def generic_batch_device(monkeypatch):
    from fuzzysearch_b200 import search
    monkeypatch.setattr(F, "Haystack", GenericBatchHaystack)
    monkeypatch.setattr(F, "PinnedBuffer", FakePinnedBuffer)
    monkeypatch.setattr(F, "device_count", lambda: 1)
    saved = dict(search._WORKSPACE)
    search._WORKSPACE.clear()
    del CALLS[:]
    yield
    search._WORKSPACE.clear()
    search._WORKSPACE.update(saved)


SEQ = b"xxGATTACAxxGATTTCAxxGATACAxxCATTACAGxxGATTACAxxGATTAACAxx" * 3
PATS = [b"GATTACA", b"GATTTCA", b"CATTACAG", b"GATTACA", b"ATTAC", b"GATTAACA"]
LIMITS = [dict(max_substitutions=1, max_insertions=1, max_deletions=0, max_l_dist=1),   # generic
          dict(max_l_dist=1),                                                           # Levenshtein
          dict(max_substitutions=0, max_insertions=1, max_deletions=1),                 # generic, total = 2
          dict(max_substitutions=2, max_insertions=0, max_deletions=0),                 # substitutions only
          dict(max_substitutions=5, max_insertions=1, max_deletions=0, max_l_dist=2),   # generic, subs -> 2
          dict(max_substitutions=1, max_insertions=0, max_deletions=1, max_l_dist=9)]   # generic, total -> 2


def per_pattern(limits):
    return {key: [d.get(key) for d in limits]
            for key in ("max_substitutions", "max_insertions", "max_deletions", "max_l_dist")}


def test_generic_patterns_take_the_generic_batch(generic_batch_device):
    got = find_near_matches_batch(PATS, SEQ, **per_pattern(LIMITS))
    assert got == [find_near_matches(p, SEQ, **d) for p, d in zip(PATS, LIMITS)]
    assert all(got)
    batch_calls = [c for c in CALLS if c[0].endswith("_batch")]
    assert batch_calls == [
        ("levenshtein_batch", [PATS[1]], [1]),
        ("hamming_batch", [PATS[3]], [2]),
        # input order, limits normalised as LevenshteinSearchParams does
        ("generic_batch", [PATS[0], PATS[2], PATS[4], PATS[5]], [(1, 1, 0, 1), (0, 1, 1, 2), (2, 1, 0, 2),
                                                                  (1, 0, 1, 2)])]


def test_one_limit_for_every_pattern(generic_batch_device):
    kw = dict(max_substitutions=1, max_insertions=1, max_deletions=0, max_l_dist=2)
    got = find_near_matches_batch(PATS, SEQ, **kw)
    assert got == [find_near_matches(p, SEQ, **kw) for p in PATS]
    first = [c for c in CALLS if c[0] == "generic_batch"][0]
    assert first == ("generic_batch", PATS, [(1, 1, 0, 2)] * len(PATS))


def test_a_single_generic_pattern_runs_on_its_own(generic_batch_device):
    got = find_near_matches_batch(PATS[:2], SEQ, **per_pattern(LIMITS[:2]))
    assert got == [find_near_matches(p, SEQ, **d) for p, d in zip(PATS[:2], LIMITS[:2])]
    assert ("generic", PATS[0], (1, 1, 0, 1)) in CALLS
    assert "generic_batch" not in [c[0] for c in CALLS]
