"""fuzzysearch_b200 -- H100-native (sm_90a CUDA) drop-in for fuzzysearch's near-match search.

Same public API as the reference (fuzzysearch/__init__.py:35-83):

>>> find_near_matches(b'PATTERN', b'---PATERN---', max_l_dist=1)
[Match(start=3, end=9, dist=1, matched=b'PATERN')]

Every search runs as hand-written CUDA kernels behind the C-ABI of libfuzzb200.so
(include/fuzzb200.h); there is no CPU fallback -- without the library or a GPU the calls raise.
"""
__version__ = "0.1.0"

__all__ = ["find_near_matches", "find_near_matches_batch", "find_near_matches_in_each",
           "find_near_matches_batch_in_each", "best_match_in_each", "BestMatches", "find_near_matches_in_file",
           "nearest_distance", "find_nearest_matches", "nearest_distance_in_each", "NearestDistances",
           "nearest_distance_batch", "find_nearest_matches_batch", "nearest_pattern_in_each", "NearestPatterns",
           "align_matches", "align_in_each", "Alignments", "has_near_match", "Match", "LevenshteinSearchParams", "DeviceSequence", "DeviceSequenceSet", "ExactSearch", "SubstitutionsOnlySearch", "LevenshteinSearch",
           "GenericSearch", "choose_search_class", "search_exact"]

from .common import LevenshteinSearchParams, Match
from .search import (DeviceSequence, ExactSearch, GenericSearch, LevenshteinSearch,
                     SubstitutionsOnlySearch, find_nearest_matches, find_nearest_matches_batch,
                     align_matches, nearest_distance, nearest_distance_batch, search_exact)
from .sequence_set import (Alignments, BestMatches, DeviceSequenceSet, NearestDistances, NearestPatterns, best_match_in_each,
                           find_near_matches_batch_in_each, find_near_matches_in_each, nearest_distance_in_each,
                           align_in_each, nearest_pattern_in_each)


def find_near_matches(subsequence, sequence, max_substitutions=None, max_insertions=None,
                      max_deletions=None, max_l_dist=None):
    """search for near-matches of subsequence in sequence (fuzzysearch/__init__.py:35-57).

    The nearly-matching parts of the sequence must meet the given limits on substitutions,
    insertions, deletions and their total (the Levenshtein distance)."""
    search_params = LevenshteinSearchParams(max_substitutions, max_insertions, max_deletions,
                                            max_l_dist)
    search_class = choose_search_class(search_params)
    matches = search_class.search(subsequence, sequence, search_params)
    return search_class.consolidate_matches(matches)


def has_near_match(subsequence, sequence, max_substitutions=None, max_insertions=None, max_deletions=None,
                   max_l_dist=None):
    """True iff find_near_matches(...) would return at least one match -- the public-API form of the
    reference's internal has_near_match_* helpers (substitutions_only.py:18-34,139-145,218-233;
    generic_search.py:240-253), with early termination: the sequence is searched in chunks of growing size and
    the call returns after the first chunk that holds a match (fzb_has_near_match)."""
    from .search import _lock_for, _normalised_limits, _prepare
    search_params = LevenshteinSearchParams(max_substitutions, max_insertions, max_deletions, max_l_dist)
    if len(subsequence) == 0:
        raise ValueError("Given subsequence is empty!")
    with _lock_for(sequence):
        pat, hay, _ = _prepare(subsequence, sequence)
        return hay.has_near_match(pat, *_normalised_limits(search_params))


def find_near_matches_batch(subsequences, sequence, max_l_dist=None, *, max_substitutions=None,
                            max_insertions=None, max_deletions=None):
    """Many patterns over one sequence (uploaded once): -> list of find_near_matches(...) results.

    Each limit is None, one int, or one value per pattern.  Equivalent to
    ``[find_near_matches(p, sequence, max_substitutions=s, max_insertions=i, max_deletions=d, max_l_dist=l)
    for p, s, i, d, l in zip(subsequences, ...)]``: exact and Levenshtein searches share passes over the
    sequence (fzb_search_levenshtein_batch), substitutions-only searches too (fzb_search_hamming_batch), and so do
    searches with other (generic) limits (fzb_search_generic_batch); all of them use the same uploaded sequence."""
    subsequences, limits, params, classes = _batch_params(subsequences, max_substitutions, max_insertions,
                                                          max_deletions, max_l_dist)
    if not subsequences:
        return []
    from .search import _bind_common, _lock_for, _prepare_many, _to_matches
    with _lock_for(sequence):
        bound = _bind_common(_prepare_many, subsequences, sequence)
        if bound is None:
            return [find_near_matches(p, sequence, *lim) for p, lim in zip(subsequences, limits)]
        pats, hay, slicer = bound
        return [_to_matches(arrays, slicer) for arrays in _search_batch(hay, pats, params, classes, 0)]


def _batch_params(subsequences, max_substitutions, max_insertions, max_deletions, max_l_dist):
    """The limits of a batch call, each None, one int or one value per pattern, validated as find_near_matches
    validates them, before anything is uploaded: -> (patterns, limit tuples, LevenshteinSearchParams, classes)."""
    subsequences = list(subsequences)
    n = len(subsequences)

    def per_pattern(name, value):
        if value is None or isinstance(value, int):
            return [value] * n
        try:
            value = list(value)
        except TypeError:  # not a limit: LevenshteinSearchParams rejects it as find_near_matches does
            return [value] * n
        if len(value) != n:
            raise ValueError("one %s per subsequence expected" % name)
        return value

    limits = list(zip(per_pattern("max_substitutions", max_substitutions),
                      per_pattern("max_insertions", max_insertions),
                      per_pattern("max_deletions", max_deletions), per_pattern("max_l_dist", max_l_dist)))
    from .search import _check_pattern
    params, classes = [], []
    for p, lim in zip(subsequences, limits):
        sp = LevenshteinSearchParams(*lim)  # same validation as find_near_matches
        cls = choose_search_class(sp)
        _check_pattern(cls, p)
        params.append(sp)
        classes.append(cls)
    return subsequences, limits, params, classes


def _search_batch(hay, pats, params, classes, flags):
    """The patterns `pats` (bound to the handle `hay`) searched by class: exact and Levenshtein patterns in one
    Levenshtein batch, substitutions-only ones in one Hamming batch, generic ones in one generic batch (a lone
    generic pattern on its own).  -> per pattern, its (start, end, dist) arrays in the list find_near_matches
    returns.  The caller holds the handle's lock."""
    from .search import _list_of, _max_substitutions, _search_one
    n = len(pats)
    results = [None] * n
    lev = [i for i in range(n) if classes[i] in (ExactSearch, LevenshteinSearch)]
    ham = [i for i in range(n) if classes[i] is SubstitutionsOnlySearch]
    gen = [i for i in range(n) if classes[i] is GenericSearch]
    try:
        if lev:
            rs, _ = hay.search_levenshtein_batch([pats[i] for i in lev], [params[i].max_l_dist for i in lev], flags)
            for i, r in zip(lev, rs):
                results[i] = r
        if ham:
            ks = [_max_substitutions(params[i]) for i in ham]
            rs, _ = hay.search_hamming_batch([pats[i] for i in ham], ks, flags)
            for i, r in zip(ham, rs):
                results[i] = r
        if len(gen) == 1:  # (nothing to share; the single search needs no flag to honour a record set)
            results[gen[0]] = _search_one(GenericSearch, hay, pats[gen[0]], params[gen[0]])[0]
        elif gen:  # the normalised limits GenericSearch.search applies
            rs, _ = hay.search_generic_batch([pats[i] for i in gen], *zip(*[params[i].unpacked for i in gen]),
                                             flags=flags)
            for i, r in zip(gen, rs):
                results[i] = r
        return [res.arrays(_list_of(cls)) for res, cls in zip(results, classes)]
    finally:
        for res in results:
            if res is not None:
                res.close()


def choose_search_class(search_params):
    """fuzzysearch/__init__.py:60-83."""
    max_substitutions, max_insertions, max_deletions, max_l_dist = search_params.unpacked
    if max_l_dist == 0:
        return ExactSearch
    elif max_insertions == 0 and max_deletions == 0:
        return SubstitutionsOnlySearch
    elif max_l_dist <= min(
            (max_substitutions if max_substitutions is not None else (1 << 29)),
            (max_insertions if max_insertions is not None else (1 << 29)),
            (max_deletions if max_deletions is not None else (1 << 29)),
    ):
        return LevenshteinSearch
    else:
        return GenericSearch


def find_near_matches_in_file(subsequence, sequence_file, max_substitutions=None, max_insertions=None,
                              max_deletions=None, max_l_dist=None, _chunk_size=2 ** 20):
    """search for near-matches of subsequence in a file (fuzzysearch/__init__.py:86-200)."""
    from .file_search import find_near_matches_in_file as impl
    return impl(subsequence, sequence_file, max_substitutions, max_insertions, max_deletions,
                max_l_dist, _chunk_size)
