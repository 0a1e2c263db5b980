"""Seeded fuzz of the CPU oracle against outputs of the REAL reference, stored in
tests/golden/ref_live_fuzz.json.  Complements ref_fuzz.json with a second case generator (longer
patterns and haystacks, every route function and the final list).

The cases are regenerated from SEED on every run; the fixture holds the reference's answers (raw streams
as digests, final lists whole where tied groups make them order-dependent, else as digests) and a digest
of the inputs they were computed for.  To regenerate it (pure-Python reference sources):

    PYTHONHASHSEED=0 PYTHONPATH=. python tests/test_oracle_live_reference.py <reference>/src
"""
import hashlib
import json
import os
import random
import sys

import oracle
from parity import GOLDEN_DIR, admissible_sets, assert_final_parity, is_admissible_final, load_golden, tup

SEED = 20261015
FIXTURE = "ref_live_fuzz.json"


def _case(rng, mmax=28, nmax=220):
    alphabet = rng.choice([b"ab", b"ACGT", b"abcdefgh", bytes(range(32, 127))])
    m = rng.randint(1, mmax)
    pat = bytes(rng.choice(alphabet) for _ in range(m))
    hay = bytearray(rng.choice(alphabet) for _ in range(rng.randint(0, nmax)))
    for _ in range(rng.randint(0, 4)):
        v = bytearray(pat)
        for _ in range(rng.randint(0, 4)):
            op = rng.randrange(3)
            if op == 0 and v:
                v[rng.randrange(len(v))] = rng.choice(alphabet)
            elif op == 1:
                v.insert(rng.randrange(len(v) + 1), rng.choice(alphabet))
            elif v:
                del v[rng.randrange(len(v))]
        pos = rng.randint(0, len(hay))
        hay[pos:pos + len(v)] = v
    return pat, bytes(hay)


def _cases():
    """-> [(kind, pattern, haystack, limits)]: "lev" cases take max_l_dist k, "generic" cases
    (max_substitutions, max_insertions, max_deletions, max_l_dist)."""
    rng = random.Random(SEED)
    out = []
    for _ in range(1500):
        pat, hay = _case(rng)
        out.append(("lev", pat, hay, (rng.randint(0, 5),)))
    for _ in range(400):
        pat, hay = _case(rng, 16, 80)
        subs, ins, dels = rng.randint(0, 3), rng.randint(0, 3), rng.randint(0, 3)
        out.append(("generic", pat, hay, (subs, ins, dels, rng.choice([None, rng.randint(0, 4)]))))
    return out


def _digest(cases):
    h = hashlib.sha256()
    for kind, pat, hay, lim in cases:
        h.update(repr((kind, pat, hay, lim)).encode())
    return h.hexdigest()


def _results_digest(named):
    """[(function name, match triples)] -> 10 hex digits: the fixture stores the reference's raw streams this way."""
    return hashlib.sha256(json.dumps([[n, [list(t) for t in tup(ms)]] for n, ms in named]).encode()).hexdigest()[:10]


def _oracle_streams(kind, pat, hay, lim, up=None):
    """The oracle's raw streams of one case, named like the reference functions they restate."""
    out = []
    if kind == "lev":
        (k,) = lim
        if len(pat) // (k + 1) >= 1:
            out.append(("lev_ngrams", oracle.levenshtein_ngrams_raw(pat, hay, k)))
            out.append(("subs_ngrams", oracle.subs_ngrams(pat, hay, k)))
        if len(pat) <= 12 and k <= 3:
            out.append(("lev_lp", oracle.levenshtein_lp_raw(pat, hay, k)))
        out.append(("subs_lp", oracle.subs_lp(pat, hay, k)))
    else:
        out.append(("generic_lp", oracle.generic_lp_raw(pat, hay, *up)))
        if len(pat) // (up[3] + 1) >= 1:
            out.append(("generic_ngrams", oracle.generic_ngrams_raw(pat, hay, *up)))
    return out


def test_live_fuzz_against_reference():
    cases = _cases()
    with open(os.path.join(GOLDEN_DIR, FIXTURE)) as f:
        assert json.load(f)["inputs_sha256"] == _digest(cases), "case generator differs from the fixture's"
    records = load_golden(FIXTURE)
    assert len(records) == len(cases)
    for (kind, pat, hay, lim), (streams, ref_final, up) in zip(cases, records):
        ctx = (pat, hay, lim)
        if kind == "generic":
            assert list(oracle.normalize_params(*lim)) == up, ctx
        assert _results_digest(_oracle_streams(kind, pat, hay, lim, up)) == streams, ctx
        if kind == "lev" and lim[0] > 0:
            final, raw = oracle.find_near_matches(pat, hay, max_l_dist=lim[0], return_raw=True)
            if isinstance(ref_final, list):
                assert_final_parity(final, ref_final, raw, repr(ctx))
            else:
                assert _results_digest([("final", final)]) == ref_final, ctx
                assert is_admissible_final(final, raw), ctx


def _record(ref_src):
    """Runs every case through the reference's pure-Python functions and writes the fixture."""
    sys.path.insert(0, ref_src)
    import fuzzysearch
    from fuzzysearch import generic_search, levenshtein, levenshtein_ngram, substitutions_only
    from fuzzysearch.common import LevenshteinSearchParams

    def t(ms):
        return [[m.start, m.end, m.dist] for m in ms]

    cases = _cases()
    records = []
    for kind, pat, hay, lim in cases:
        streams, final, up = [], None, None
        if kind == "lev":
            (k,) = lim
            if len(pat) // (k + 1) >= 1:
                streams.append(("lev_ngrams", t(levenshtein_ngram.find_near_matches_levenshtein_ngrams(pat, hay, k))))
                streams.append(("subs_ngrams", t(substitutions_only.find_near_matches_substitutions_ngrams(pat, hay, k))))
            if len(pat) <= 12 and k <= 3:
                streams.append(("lev_lp", t(levenshtein.find_near_matches_levenshtein_linear_programming(pat, hay, k))))
            streams.append(("subs_lp", t(substitutions_only.find_near_matches_substitutions_lp(pat, hay, k))))
            if k > 0:
                # the winner of a group with tied minimisers depends on set order: such lists are stored whole
                final = t(fuzzysearch.find_near_matches(pat, hay, max_l_dist=k))
                raw = oracle.find_near_matches(pat, hay, max_l_dist=k, return_raw=True)[1]
                if all(len(g) == 1 for g in admissible_sets(raw)):
                    final = _results_digest([("final", final)])
        else:
            params = LevenshteinSearchParams(*lim)
            up = list(params.unpacked)
            streams.append(("generic_lp", t(generic_search._find_near_matches_generic_linear_programming(pat, hay, params))))
            if len(pat) // (up[3] + 1) >= 1:
                streams.append(("generic_ngrams", t(generic_search.find_near_matches_generic_ngrams(pat, hay, params))))
        records.append([_results_digest(streams), final, up])
    out = {"source": "tests/test_oracle_live_reference.py cases (random.Random(%d)) through the pure-Python "
                     "reference (fuzzysearch 0.8.1), PYTHONHASHSEED=0" % SEED,
           "inputs_sha256": _digest(cases), "records": records}
    with open(os.path.join(GOLDEN_DIR, FIXTURE), "w") as f:
        json.dump(out, f, separators=(",", ":"))
    print("%d records -> %s" % (len(records), FIXTURE))


if __name__ == "__main__":
    _record(sys.argv[1])
