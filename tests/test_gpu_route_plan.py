"""One plan per pattern (api.cu, plan_*): the single searches, their batches and fzb_best_per_record refuse a pattern
with one and the same error and leave the handle usable, and a generic pattern whose max_l_dist is far above its
length (2^32 - 1 included) runs the generic LP route with the lowered limit m + max_insertions."""
import numpy as np
import pytest

import oracle
from fuzzysearch_b200 import _native as F, best_match_in_each, find_near_matches, has_near_match
from parity import tup
from test_gpu_best_match import assert_columns, oracle_lists, reduce_lists
from test_gpu_records import joined

pytestmark = pytest.mark.gpu

BIG = 2**32 - 1
TEXT = (b"the quick brown fox jumps over the lazy dog; abcdef abXdef abcdf abcxdef pack my box with five dozen "
        b"liquor jugs. ") * 40

# class -> (valid pattern and limits (subs, ins, dels, max_l), single(hs, p, lim, flags), batch(hs, pats, lims, flags))
CLASSES = {
    "levenshtein": ((b"quick", (1, 1, 1, 1)), lambda hs, p, l, f: hs.search_levenshtein(p, l[3], f),
                    lambda hs, ps, ls, f: hs.search_levenshtein_batch(ps, [l[3] for l in ls], f)),
    "hamming": ((b"quick", (1, 0, 0, 1)), lambda hs, p, l, f: hs.search_hamming(p, l[0], f),
                lambda hs, ps, ls, f: hs.search_hamming_batch(ps, [l[0] for l in ls], f)),
    "generic": ((b"quick", (1, 1, 0, 2)), lambda hs, p, l, f: hs.search_generic(p, *l, f),
                lambda hs, ps, ls, f: hs.search_generic_batch(ps, *zip(*ls), flags=f)),
    "exact": ((b"quick", (0, 0, 0, 0)), lambda hs, p, l, f: hs.search_exact(p, f), None),
}

# (refusal, class, pattern, limits, flags, handle): "shard" is an interior shard whose buffer reaches 16 bytes past
# its own range on each side; fzb_best_per_record takes no flags and no shard, so it joins where both are plain
REFUSALS = [(name, cls, p, CLASSES[cls][0][1], 0, "whole")
            for cls in CLASSES for name, p in (("empty", b""), ("256 symbols", b"q" * 256))]
REFUSALS += [("shard halo", cls, b"the quick brown fox jumps", CLASSES[cls][0][1], 0, "shard") for cls in CLASSES]
REFUSALS += [
    ("max_l_dist > 63", "generic", b"the quick brown fox ", (100, 64, 64, 100), 0, "whole"),
    ("n-gram length 0", "levenshtein", b"ab", (2, 2, 2, 2), F.F_FORCE_NGRAMS, "whole"),
    ("n-gram length 0", "generic", b"ab", (1, 1, 1, 2), F.F_FORCE_NGRAMS, "whole"),
]
REFUSALS += [("FZB_F_GLOBAL without a world", cls, b"quick", CLASSES[cls][0][1], F.F_GLOBAL, "whole")
             for cls in ("levenshtein", "hamming", "generic")]


def raw_rows(r):
    return list(zip(*[a.tolist() for a in r.arrays(F.RAW, anchors=True)]))


def lists(r):
    return raw_rows(r), r.triples(F.FINAL), r.group_rows().tolist()


def refusal(call):
    with pytest.raises(Exception) as e:
        call()
    return type(e.value), str(e.value)


def test_one_refusal_for_the_single_search_its_batch_and_best_per_record(cuda_device):
    hay = np.frombuffer(TEXT, dtype=np.uint8).copy()
    n, lo, hi = len(hay), 1024, 2048
    handles = {"whole": F.Haystack.from_host(hay),
               "shard": F.Haystack.from_host(hay[lo - 16:hi + 16], buf_lo=lo - 16, global_len=n, own_lo=lo, own_hi=hi)}
    buf, off = joined([TEXT[j:j + 299] for j in range(0, n, 300)])
    recs = F.Haystack.from_host(np.frombuffer(buf, dtype=np.uint8).copy())
    recs.set_records(off)
    valid = [CLASSES[c][0] for c in CLASSES]
    vpats, vlims = [p for p, _ in valid], [l for _, l in valid]

    def usable(hs):  # every class's single search, and the Levenshtein batch, still work and agree
        out = [lists(CLASSES[c][1](hs, p, l, 0)) for c, (p, l) in zip(CLASSES, valid)]
        rs, _ = hs.search_levenshtein_batch(vpats, [1] * len(vpats))
        return out + [lists(r) for r in rs]

    before = {k: usable(hs) for k, hs in handles.items()}
    best_before, _ = recs.best_per_record(vpats, *zip(*vlims))
    for name, cls, p, lim, flags, where in REFUSALS:
        ctx = (name, cls)
        hs = handles[where]
        (_, vlim), single, batch = CLASSES[cls]
        want = refusal(lambda: single(hs, p, lim, flags))
        assert want[0] in (ValueError, F.UnsupportedError), ctx + want
        if batch is not None:  # the refused pattern after valid ones of its class
            assert refusal(lambda: batch(hs, vpats + [p], [vlim] * len(vpats) + [lim], flags)) == want, ctx
        if flags == 0 and where == "whole":
            bp, bl = vpats + [p], vlims + [lim]
            assert refusal(lambda: recs.best_per_record(bp, *zip(*bl))) == want, ctx
        assert usable(hs) == before[where], ctx
    got, _ = recs.best_per_record(vpats, *zip(*vlims))
    for a, b in zip(got, best_before):
        assert a.tolist() == b.tolist()
    for hs in list(handles.values()) + [recs]:
        hs.close()


# (pattern, subs, ins, dels): generic patterns whose max_l_dist = 2^32 - 1 is lowered to m + ins on the LP route
UNBOUNDED = [(b"abcdef", 1, 1, 1), (b"abcxdef", BIG, 1, 1), (b"quick", 2, 0, 1), (b"lazy dog", 1, 2, 0),
             (b"zzzzqqq", 1, 1, 1)]


def lowered(p, s, i, d):
    k = len(p) + i
    return min(s, k), i, d, k


def limits(lims):
    return dict(zip(("max_substitutions", "max_insertions", "max_deletions", "max_l_dist"), map(list, zip(*lims))))


def matches(ms):
    return [(m.start, m.end, m.dist) for m in ms]


def test_unbounded_total_limit_runs_the_lowered_lp_route(cuda_device):
    hay = np.frombuffer(TEXT, dtype=np.uint8).copy()
    hs = F.Haystack.from_host(hay)
    pats = [u[0] for u in UNBOUNDED]
    big = [(s, i, d, BIG) for _, s, i, d in UNBOUNDED]
    low = [lowered(*u) for u in UNBOUNDED]
    many, _ = hs.search_generic_batch(pats, *zip(*big))
    for p, b, l, r in zip(pats, big, low, many):
        one, ref = hs.search_generic(p, *b), hs.search_generic(p, *l)
        assert one.stats()["route"] == ref.stats()["route"] == "generic-lp", p
        assert lists(one) == lists(ref) == lists(r), p
        assert sorted(one.triples(F.RAW)) == sorted(tup(oracle.generic_raw(p, TEXT, *l))), p
        kw = dict(max_substitutions=b[0], max_insertions=b[1], max_deletions=b[2])
        fin = matches(find_near_matches(p, TEXT, max_l_dist=BIG, **kw))
        assert fin == matches(find_near_matches(p, TEXT, max_l_dist=l[3], **kw)), p
        assert fin == tup(oracle.find_near_matches(p, TEXT, *l)), p
        assert has_near_match(p, TEXT, max_l_dist=BIG, **kw) == bool(fin), p
        for x in (one, ref, r):
            x.close()
    hs.close()
    # one row per record: the binding with the raw limits, and best_match_in_each
    seqs = [TEXT[j:j + 97] for j in range(0, 2000, 97)]
    buf, off = joined(seqs)
    rec = F.Haystack.from_host(np.frombuffer(buf, dtype=np.uint8).copy())
    rec.set_records(off)
    got, _ = rec.best_per_record(pats, *zip(*big))
    ref, _ = rec.best_per_record(pats, *zip(*low))
    for a, b in zip(got, ref):
        assert a.tolist() == b.tolist()
    rec.close()
    exp = reduce_lists(oracle_lists(pats, seqs, limits(low), range(len(seqs))), len(seqs))
    assert_columns(best_match_in_each(pats, seqs, **limits(big)), exp)
    assert_columns(best_match_in_each(pats, seqs, **limits(low)), exp)
    assert_columns(got, exp)
