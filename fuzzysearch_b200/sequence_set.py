"""One pattern over many sequences in one device pass: ``find_near_matches_in_each`` and ``DeviceSequenceSet``.

The sequences are joined into one resident buffer, each followed by one separator position, and the buffer is
declared a record set (fzb_haystack_set_records, DESIGN.md section 5.10): the kernels clip every window at the edges
of the record it belongs to, so one search returns, in buffer coordinates, what searching each sequence alone would
return.  The lists are split per sequence on the host by the start of each match."""
import threading

import numpy as np

from . import _native
from .common import LevenshteinSearchParams, Match
from .search import (_BIG, DeviceSequence, _bind_common, _check_pattern, _kind, _matches, _nearest_flags,
                     _normalised_limits, _search_one, _slicer, _text)

__all__ = ["Alignments", "BestMatches", "DeviceSequenceSet", "NearestDistances", "NearestPatterns", "align_in_each",
           "best_match_in_each",
           "find_near_matches_in_each", "find_near_matches_batch_in_each", "nearest_distance_in_each",
           "nearest_pattern_in_each"]


def _set_kind(sequences):
    """'str' | 'bytes' for a list of sequences of one kind (Bio.Seq.Seq counts as str)."""
    kinds = set()
    for s in sequences:
        k = _kind(_text(s))
        if k == "items":
            raise TypeError("sequences of items (lists / tuples) are not supported in a sequence set")
        kinds.add(k)
    if len(kinds) > 1:
        raise TypeError("the sequences of a set must all be str or all be byte-like")
    return kinds.pop() if kinds else "bytes"


class DeviceSequenceSet(object):
    """Many sequences kept resident in HBM as one record set, searched with any number of patterns by
    ``find_near_matches_in_each(pattern, this_set, ...)``.  ``len()`` is the number of sequences."""

    def __init__(self, sequences, device=0):
        if not isinstance(sequences, (list, tuple)):
            raise TypeError("sequences must be a list or tuple")
        self._lock = threading.RLock()
        self._orig = list(sequences)
        self._kind = _set_kind(self._orig)
        texts = [_text(s) for s in self._orig]
        lengths = np.fromiter((len(t) for t in texts), dtype=np.uint64, count=len(texts))
        self.offsets = np.zeros(len(texts) + 1, dtype=np.uint64)
        np.cumsum(lengths + 1, out=self.offsets[1:])
        if self._kind == "str":
            joined = "\0".join(texts) + "\0"
        else:
            # byte-like elements go through as_u8: the single-byte, contiguous check find_near_matches applies
            joined = b"\0".join(t if isinstance(t, (bytes, bytearray)) else _native.as_u8(t) for t in texts) + b"\0"
        self._seq = DeviceSequence(joined, device=device)
        self._bound_alphabet = self._seq._alphabet
        self._seq.haystack.set_records(self.offsets)

    def __len__(self):
        return len(self._orig)

    def _bind(self, subsequence):
        return self._bind_many([subsequence])[0]

    def _bind_many(self, subsequences):
        """-> the patterns in the resident set's byte alphabet; a re-reduction of a wide-symbol set (a new upload,
        which clears the record set) is followed by declaring the records again."""
        pats = self._seq._bind_many(subsequences)
        if self._seq._alphabet != self._bound_alphabet:
            self._seq.haystack.set_records(self.offsets)
            self._bound_alphabet = self._seq._alphabet
        return pats

    def close(self):
        self._seq.close()


def _check_sequences(sequences):
    if not isinstance(sequences, (DeviceSequenceSet, list, tuple)):
        raise TypeError("sequences must be a list, a tuple or a DeviceSequenceSet")


def _in_each(sequences, empty, body):
    """The frame of the *_in_each calls: -> body(seqset) on a resident set -- `sequences` itself, or one uploaded from
    the list / tuple for this call and closed on every exit -- or empty(sequences), uploading nothing, when there is
    nothing to do: no sequences, or no body (nothing to search for)."""
    _check_sequences(sequences)
    if body is None or len(sequences) == 0:
        return empty(sequences)
    if isinstance(sequences, DeviceSequenceSet):
        return body(sequences)
    seqset = DeviceSequenceSet(sequences)
    try:
        return body(seqset)
    finally:
        seqset.close()


def find_near_matches_in_each(subsequence, sequences, max_substitutions=None, max_insertions=None,
                              max_deletions=None, max_l_dist=None):
    """One pattern over many sequences: -> a list with, for every sequence, exactly
    ``find_near_matches(subsequence, sequences[i], ...)``.  `sequences` is a list / tuple (uploaded for this call)
    or a DeviceSequenceSet (resident).  All of them are searched in one device pass.  The limits are validated once
    for the call, before anything else (also when there are no sequences)."""
    search_params = LevenshteinSearchParams(max_substitutions, max_insertions, max_deletions, max_l_dist)
    from . import choose_search_class
    cls = choose_search_class(search_params)
    _check_pattern(cls, subsequence)
    return _in_each(sequences, lambda _: [], lambda seqset: _search_set(subsequence, seqset, cls, search_params))


def _search_set(subsequence, seqset, cls, search_params):
    with seqset._lock:
        res, which = _search_one(cls, seqset._seq.haystack, seqset._bind(subsequence), search_params)
        try:
            s, e, d = res.arrays(which)
        finally:
            res.close()
    out = [[] for _ in range(len(seqset))]
    for i, matches in _split_by_record(seqset, s, e, d):
        out[i] = matches
    return out


def _split_by_record(seqset, s, e, d):
    """One search's list over the set (buffer coordinates) -> (sequence index, its Match list) for every sequence
    that holds matches, in sequence order; positions relative to the sequence, `matched` sliced from it."""
    offsets = seqset.offsets.astype(np.int64)
    rec = np.searchsorted(offsets, s, side="right") - 1
    order = np.argsort(rec, kind="stable")  # each record's matches keep their order
    rec, s, e, d = rec[order], s[order], e[order], d[order]
    base = offsets[rec]
    s, e, d = (s - base).tolist(), (e - base).tolist(), d.tolist()
    # only the records that hold matches are visited (most short sequences hold none)
    hit_recs, firsts = np.unique(rec, return_index=True)
    ends = np.append(firsts[1:], len(s))
    for i, lo, hi in zip(hit_recs.tolist(), firsts.tolist(), ends.tolist()):
        yield i, _matches(s[lo:hi], e[lo:hi], d[lo:hi], _slicer(seqset._orig[i], seqset._kind))


def find_near_matches_batch_in_each(subsequences, sequences, max_l_dist=None, *, max_substitutions=None,
                                    max_insertions=None, max_deletions=None):
    """Many patterns over many sequences: -> one dict per pattern, mapping the index of every sequence that holds
    matches to its non-empty list, so that ``out[i].get(r, []) == find_near_matches(subsequences[i], sequences[r],
    ...)``.  The limits are taken as find_near_matches_batch takes them (None, one int, or one value per pattern)
    and validated before anything is uploaded.  `sequences` is a list / tuple (uploaded for this call) or a
    DeviceSequenceSet (resident).  The patterns share passes over the whole set as in find_near_matches_batch
    (fzb_search_*_batch with FZB_F_PER_RECORD, DESIGN.md section 5.11)."""
    from . import _batch_params
    subsequences, limits, params, classes = _batch_params(subsequences, max_substitutions, max_insertions,
                                                          max_deletions, max_l_dist)
    if not subsequences:
        return []
    return _in_each(sequences, lambda _: [{} for _ in subsequences],
                    lambda seqset: _search_set_batch(subsequences, seqset, limits, params, classes))


def _search_set_batch(subsequences, seqset, limits, params, classes):
    from . import _search_batch
    with seqset._lock:
        pats = _bind_common(seqset._bind_many, subsequences)
        if pats is not None:
            lists = _search_batch(seqset._seq.haystack, pats, params, classes, _native.F_PER_RECORD)
    if pats is None:
        return [dict((r, ms) for r, ms in enumerate(find_near_matches_in_each(p, seqset, *lim)) if ms)
                for p, lim in zip(subsequences, limits)]
    return [dict(_split_by_record(seqset, s, e, d)) for s, e, d in lists]


class BestMatches(object):
    """What best_match_in_each returns: six numpy arrays with one entry per sequence, -1 where a sequence holds no
    match.  ``pattern``: the index of the nearest pattern (the smallest index among equals); ``dist``, ``start``,
    ``end``: its best match there (the smallest distance, then the longest, then the leftmost), in the sequence's own
    coordinates; ``second_pattern``, ``second_dist``: the nearest match of any OTHER pattern (the smallest index
    among equals), for rejecting ambiguous calls by ``second_dist - dist``.  ``best[r]`` is None or
    ``(pattern index, Match)``, the Match built (and its ``matched`` sliced from the sequence) when asked for."""

    def __init__(self, sequences, kind, columns):
        self._sequences, self._kind = sequences, kind
        self.pattern, self.start, self.end, self.dist, self.second_pattern, self.second_dist = columns

    def __len__(self):
        return len(self.pattern)

    def __getitem__(self, r):
        if self.pattern[r] < 0:
            return None
        s, e = int(self.start[r]), int(self.end[r])
        matched = _slicer(self._sequences[r], self._kind)(s, e)
        return int(self.pattern[r]), Match(s, e, int(self.dist[r]), matched=matched)


def _no_matches(n):
    return tuple(np.full(n, -1, dtype=t) for t in (np.int32, np.int64, np.int64, np.int32, np.int32, np.int32))


def best_match_in_each(subsequences, sequences, max_l_dist=None, *, max_substitutions=None, max_insertions=None,
                       max_deletions=None):
    """Many patterns over many sequences, reduced on the device to one row per sequence: -> BestMatches, the
    nearest pattern of every sequence, its best match there and the runner-up among the other patterns -- what
    reducing ``find_near_matches_batch_in_each(...)`` over the patterns gives, without building its lists
    (fzb_best_per_record, DESIGN.md section 5.13).  Patterns, limits and `sequences` are taken and validated as
    find_near_matches_batch_in_each takes them."""
    from . import _batch_params
    subsequences, limits, params, classes = _batch_params(subsequences, max_substitutions, max_insertions,
                                                          max_deletions, max_l_dist)

    def no_rows(seqs):
        orig = seqs._orig if isinstance(seqs, DeviceSequenceSet) else list(seqs)
        return BestMatches(orig, _set_kind(orig), _no_matches(len(orig)))
    return _in_each(sequences, no_rows, (lambda seqset: _best_in_set(subsequences, seqset, limits, params))
                    if subsequences else None)


def _best_in_set(subsequences, seqset, limits, params):
    with seqset._lock:
        pats = _bind_common(seqset._bind_many, subsequences)
        if pats is not None:
            lims = zip(*[_normalised_limits(p) for p in params])
            columns, _ = seqset._seq.haystack.best_per_record(pats, *lims)
    if pats is None:
        columns = _best_on_host(subsequences, seqset, limits)
    return BestMatches(seqset._orig, seqset._kind, columns)


def _best_on_host(subsequences, seqset, limits):
    """The same rows from find_near_matches_in_each, pattern by pattern (each reduces the set to its own alphabet)."""
    pat, start, end, dist, pat2, dist2 = columns = _no_matches(len(seqset))
    for i, (p, lim) in enumerate(zip(subsequences, limits)):
        d, s, e = np.full(len(seqset), -1, dtype=np.int32), np.full(len(seqset), -1), np.full(len(seqset), -1)
        for r, matches in enumerate(find_near_matches_in_each(p, seqset, *lim)):
            if matches:
                m = min(matches, key=lambda x: (x.dist, x.start - x.end, x.start))
                d[r], s[r], e[r] = m.dist, m.start, m.end
        _fold(i, d, (pat, dist, pat2, dist2), ((start, s), (end, e)))
    return columns


def _fold(i, dist, columns, carried):
    """Fold pattern i's distance to every record (-1: none there) into the (pattern, dist, second_pattern,
    second_dist) columns: a strictly smaller distance replaces the winner, which becomes the runner-up; an equal one
    leaves the earlier (smaller) index in place.  carried: (column, pattern i's values) pairs that go with the
    winner."""
    pattern, best, pat2, dist2 = columns
    has = dist >= 0
    first = has & ((pattern < 0) | (dist < best))
    second = has & ~first & ((pat2 < 0) | (dist < dist2))
    pat2[first], dist2[first] = pattern[first], best[first]
    pattern[first], best[first] = i, dist[first]
    for column, values in carried:
        column[first] = values[first]
    pat2[second], dist2[second] = i, dist[second]


class NearestDistances(object):
    """What nearest_distance_in_each and nearest_distance_batch return: ``dist`` (int32) and ``end`` (int64), one
    entry per sequence (nearest_distance_in_each) or per pattern (nearest_distance_batch) -- the smallest Levenshtein
    distance of the pattern to any substring of the sequence and the first end position (in the sequence's own
    coordinates) of a substring at that distance.  ``nearest[i]`` is ``(dist, end)``.  With
    ``substitutions_only=True`` ``dist`` is the smallest number of substitutions of a window of the pattern's length,
    the match starts at ``end - len(pattern)``, and a sequence shorter than the pattern (or a pattern longer than the
    sequence) gives ``(-1, -1)``.

    ``start`` (int64) is None, except for anchored results (``anchor='start'`` / ``'end'``), where it holds the
    match's start on every row with a distance (-1 elsewhere): 0 for ``'start'``, and for ``'end'`` the largest start
    at that distance, the match then ending at the sequence's end."""

    def __init__(self, dist, end, start=None):
        self.dist, self.end, self.start = dist, end, start

    def __len__(self):
        return len(self.dist)

    def __getitem__(self, r):
        return int(self.dist[r]), int(self.end[r])


def _anchored_span(seqset, flags, has, pos):
    """The (start, end) columns of anchored rows in the sequences' own coordinates from the call's per-record
    position (the end under 'start', the start under 'end'); -1 where a row has no distance.  Unanchored: (None,
    pos)."""
    if not flags & (_native.F_ANCHOR_START | _native.F_ANCHOR_END):
        return None, pos
    if flags & _native.F_ANCHOR_START:
        return np.where(has, 0, -1).astype(np.int64), pos
    n = np.diff(seqset.offsets.astype(np.int64)) - 1
    return pos, np.where(has, n, -1).astype(np.int64)


def _no_distances(flags):
    anchored = flags & (_native.F_ANCHOR_START | _native.F_ANCHOR_END)
    return NearestDistances(np.zeros(0, np.int32), np.zeros(0, np.int64), np.zeros(0, np.int64) if anchored else None)


def nearest_distance_in_each(subsequence, sequences, *, substitutions_only=False, anchor=None):
    """One pattern over many sequences, without a distance limit: -> NearestDistances with, for every sequence,
    ``nearest_distance(subsequence, sequences[r])`` and where the nearest match first ends; an empty sequence gives
    ``(len(subsequence), 0)``.  All sequences are scanned in one device pass (fzb_nearest_per_record, DESIGN.md
    section 5.14).  `sequences` is a list / tuple (uploaded for this call) or a DeviceSequenceSet (resident).  With
    ``substitutions_only=True`` the distances are ``nearest_distance(..., substitutions_only=True)``, and a sequence
    shorter than the pattern gives ``(-1, -1)`` (DESIGN.md section 5.16).

    ``anchor='start'`` takes only matches that start at the sequence's first symbol: ``dist`` is the smallest
    ``lev(subsequence, seq[0:e])``, ``end`` the smallest such e, ``start`` 0.  ``anchor='end'`` takes only matches
    that end at its last symbol: the smallest ``lev(subsequence, seq[s:])``, ``start`` the largest such s, ``end``
    ``len(seq)``.  Under ``substitutions_only=True`` the window is the first (last) ``len(subsequence)`` symbols.
    An anchored scan reads at most ``2 * len(subsequence)`` symbols of a sequence (DESIGN.md section 5.18)."""
    if len(subsequence) == 0:
        raise ValueError("Given subsequence is empty!")
    flags = _nearest_flags(substitutions_only, anchor)
    return _in_each(sequences, lambda _: _no_distances(flags),
                    lambda seqset: _nearest_in_set(subsequence, seqset, flags))


def _nearest_in_set(subsequence, seqset, flags):
    with seqset._lock:
        pat = seqset._bind(subsequence)
        dist, end, _ = seqset._seq.haystack.nearest_per_record(pat, flags)
    start, end = _anchored_span(seqset, flags, dist >= 0, end)
    return NearestDistances(dist, end, start)


class NearestPatterns(object):
    """What nearest_pattern_in_each returns: five numpy arrays with one entry per sequence.  ``dist`` (int32): the
    smallest nearest_distance of any pattern to the sequence; ``pattern`` (int32): the smallest index of a pattern at
    that distance; ``end`` (int64): where its nearest match first ends, in the sequence's own coordinates (the end
    nearest_distance_in_each gives for it); ``second_pattern``, ``second_dist`` (int32): the same over the OTHER
    patterns, for rejecting ambiguous calls by ``second_dist - dist``.  Every pattern has a distance (at most its
    length), so -1 appears only in the ``second_*`` arrays with a single pattern and everywhere with none.
    ``nearest[r]`` is ``(pattern, dist, end)``.

    With ``substitutions_only=True`` only the patterns that fit in the sequence (``len(pattern) <= len(sequence)``)
    have a distance and take part: a row where none fits is -1 everywhere, one where a single pattern fits has -1 in
    the ``second_*`` arrays.  The winner's match starts at ``end - len(subsequences[pattern])``.

    ``start`` (int64) is None, except for anchored results, where it holds the winner's match start on every row
    with a pattern (-1 elsewhere), as NearestDistances.start does."""

    def __init__(self, columns, start=None):
        self.pattern, self.dist, self.end, self.second_pattern, self.second_dist = columns
        self.start = start

    def __len__(self):
        return len(self.pattern)

    def __getitem__(self, r):
        return int(self.pattern[r]), int(self.dist[r]), int(self.end[r])


def _no_patterns(n):
    return tuple(np.full(n, -1, dtype=t) for t in (np.int32, np.int32, np.int64, np.int32, np.int32))


def _no_patterns_rows(n, flags):
    anchored = flags & (_native.F_ANCHOR_START | _native.F_ANCHOR_END)
    return NearestPatterns(_no_patterns(n), np.full(n, -1, dtype=np.int64) if anchored else None)


def nearest_pattern_in_each(subsequences, sequences, *, substitutions_only=False, anchor=None):
    """Many patterns over many sequences, without a distance limit: -> NearestPatterns, for every sequence the
    pattern nearest to it, its distance and first end, and the runner-up among the other patterns -- what reducing
    ``nearest_distance_in_each(p, sequences)`` over the patterns gives (ties to the smallest index), in shared scans
    of all sequences with the reduction on the device (fzb_nearest_best_per_record, DESIGN.md section 5.15).  An
    empty sequence gives the shortest pattern (the smallest index among equals), its length and the end 0.
    `sequences` is a list / tuple (uploaded for this call) or a DeviceSequenceSet (resident).  With
    ``substitutions_only=True`` the same over ``nearest_distance_in_each(p, sequences, substitutions_only=True)``,
    where a pattern longer than a sequence has no distance there (DESIGN.md section 5.16).  With ``anchor='start'``
    or ``'end'`` the same over ``nearest_distance_in_each(p, sequences, ..., anchor=anchor)``, the winner's match
    spanning ``[start, end)`` (DESIGN.md section 5.18): the barcode at a fixed end of a read."""
    subsequences = list(subsequences)
    if any(len(p) == 0 for p in subsequences):
        raise ValueError("Given subsequence is empty!")
    flags = _nearest_flags(substitutions_only, anchor)
    return _in_each(sequences, lambda seqs: _no_patterns_rows(len(seqs), flags),
                    (lambda seqset: _nearest_patterns_in_set(subsequences, seqset, flags)) if subsequences else None)


def _nearest_patterns_in_set(subsequences, seqset, flags):
    with seqset._lock:
        pats = _bind_common(seqset._bind_many, subsequences)
        if pats is not None:
            columns, _ = seqset._seq.haystack.nearest_best_per_record(pats, flags)
            start, end = _anchored_span(seqset, flags, columns[0] >= 0, columns[2])
            return NearestPatterns(columns[:2] + (end,) + columns[3:], start)
    columns, start = _nearest_patterns_on_host(subsequences, seqset, flags)
    return NearestPatterns(columns, start)


def _nearest_patterns_on_host(subsequences, seqset, flags):
    """The same rows from nearest_distance_in_each, pattern by pattern (each reduces the set to its own alphabet),
    and the winners' starts (None unanchored).  A pattern without a distance in a sequence (-1: substitutions only,
    longer than the sequence) is left out."""
    pattern, dist, end, pat2, dist2 = columns = _no_patterns(len(seqset))
    start = np.full(len(seqset), -1, dtype=np.int64)
    anchor = "start" if flags & _native.F_ANCHOR_START else "end" if flags & _native.F_ANCHOR_END else None
    for i, p in enumerate(subsequences):
        got = nearest_distance_in_each(p, seqset, substitutions_only=bool(flags & _native.F_SUBSTITUTIONS_ONLY),
                                       anchor=anchor)
        _fold(i, got.dist, (pattern, dist, pat2, dist2), ((end, got.end),) + (((start, got.start),) if anchor else ()))
    return columns, (start if anchor is not None else None)


class Alignments(object):
    """What align_in_each returns: numpy columns with one entry per sequence, -1 where a row has no match.  ``start``,
    ``end`` (int64): the aligned window in the sequence's own coordinates; ``dist`` (int32): the alignment's cost,
    ``substitutions + insertions + deletions``; ``cigar``: a list of extended CIGAR strings ('' for rows without a
    match).  ``al[r]`` is None or ``(start, end, cigar)``."""

    def __init__(self, columns, cigar):
        self.start, self.end, self.dist, self.substitutions, self.insertions, self.deletions = columns
        self.cigar = cigar

    def __len__(self):
        return len(self.start)

    def __getitem__(self, r):
        if self.start[r] < 0:
            return None
        return int(self.start[r]), int(self.end[r]), self.cigar[r]


def align_in_each(subsequences, sequences, rows, max_l_dist=None, *, max_substitutions=None, max_insertions=None,
                  max_deletions=None, substitutions_only=False):
    """The edit operations of one result row per sequence, aligned on the device (fzb_align, DESIGN.md section 5.17):
    -> Alignments.  `rows` is what one of these returned for the same patterns and sequences:

    * best_match_in_each: each row's match is aligned as align_matches aligns it; pass the limits it was computed
      with (taken as best_match_in_each takes them).
    * nearest_pattern_in_each / nearest_distance_in_each (one pattern): the rows give only the distance d and the end
      e; the alignment starts at the smallest s with ``lev(pattern, sequence[s:e]) == d`` -- the longest match at the
      nearest distance, found on the device from a window of at most ``len(pattern) + d`` symbols -- and its cost is
      d.  Pass the same ``substitutions_only`` (then s = e - len(pattern)); no limits.  Anchored rows (``anchor=``)
      carry their start: the window ``[start, end)`` is aligned as it is, at cost d.

    `sequences` is a list / tuple (uploaded for this call) or a DeviceSequenceSet (resident)."""
    if not isinstance(subsequences, (list, tuple)):
        subsequences = [subsequences]
    subsequences = list(subsequences)
    if any(len(p) == 0 for p in subsequences):
        raise ValueError("Given subsequence is empty!")
    n = len(rows)
    if isinstance(rows, BestMatches):
        from . import _batch_params
        subsequences, _, params, _ = _batch_params(subsequences, max_substitutions, max_insertions, max_deletions,
                                                   max_l_dist)
        lims = [_normalised_limits(p) for p in params]
        pattern, start, dist = rows.pattern, rows.start, rows.dist
        nearest = False
    else:
        if any(x is not None for x in (max_l_dist, max_substitutions, max_insertions, max_deletions)):
            raise ValueError("limits are taken only with BestMatches rows")
        lims = [(_BIG, 0, 0, _BIG) if substitutions_only else (_BIG,) * 4] * len(subsequences)  # limits that never bind
        if isinstance(rows, NearestPatterns):
            pattern = rows.pattern
        elif isinstance(rows, NearestDistances):
            if len(subsequences) != 1:
                raise ValueError("NearestDistances rows belong to one subsequence")
            pattern = np.where(rows.dist >= 0, 0, -1).astype(np.int32)
        else:
            raise TypeError("rows must be a BestMatches, NearestPatterns or NearestDistances")
        start = np.full(n, -1, dtype=np.int64) if rows.start is None else np.asarray(rows.start, dtype=np.int64)
        dist = rows.dist
        nearest = True
    _check_sequences(sequences)
    if len(sequences) != n:
        raise ValueError("one row per sequence expected")
    live = np.flatnonzero(np.asarray(pattern) >= 0)
    pidx = np.asarray(pattern)[live].astype(np.int64)
    if live.size and pidx.max() >= len(subsequences):
        raise ValueError("a row names pattern %d of %d" % (int(pidx.max()), len(subsequences)))
    cols = [np.full(n, -1, dtype=t) for t in (np.int64, np.int64, np.int32, np.int32, np.int32, np.int32)]
    cigars = [""] * n

    def align(seqset):
        base = seqset.offsets.astype(np.int64)[live]
        s = np.where(np.asarray(start)[live] >= 0, np.asarray(start)[live] + base, -1)
        e = np.asarray(rows.end)[live].astype(np.int64) + base
        d = np.asarray(dist)[live].astype(np.int32)
        (g_start, g_cost, g_x, g_ins, g_dels), cigar = _align_set(seqset, subsequences, lims, pidx, s, e, d)
        if nearest and (g_cost != d).any():
            r = int(live[np.flatnonzero(g_cost != d)[0]])
            raise RuntimeError("row %d: an alignment of cost %d at the nearest distance %d" %
                               (r, int(g_cost[np.flatnonzero(live == r)[0]]), int(dist[r])))
        ok = g_cost >= 0
        start_c, end_c, dist_c, x_c, ins_c, dels_c = cols
        rl = live[ok]
        start_c[rl] = g_start[ok] - base[ok]
        end_c[rl] = e[ok] - base[ok]
        dist_c[rl], x_c[rl], ins_c[rl], dels_c[rl] = g_cost[ok], g_x[ok], g_ins[ok], g_dels[ok]
        for r, c in zip(live.tolist(), cigar):
            cigars[r] = c
    _in_each(sequences, lambda _: None, align if live.size else None)
    return Alignments(cols, cigars)


def _align_set(seqset, subsequences, lims, pidx, s, e, d):
    """fzb_align over the set's buffer for the items (pattern pidx[i], window [s[i], e[i]) or a free start, bound
    d[i]) -> ((start, cost, substitutions, insertions, deletions) arrays, CIGAR list)."""
    from .search import _cigars
    k = len(pidx)
    cols = [np.full(k, -1, dtype=np.int64)] + [np.full(k, -1, dtype=np.int32) for _ in range(4)]
    cigar = [""] * k

    def align(sel, pats, pl, ip):  # the items `sel`, item i of pattern pats[ip[i]] with limits pl[ip[i]]
        got, ops, op_offsets, _ = seqset._seq.haystack.align(pats, *zip(*pl), ip, s[sel], e[sel], d[sel])
        for c, g in zip(cols, got):
            c[sel] = g
        m = np.array([len(p) for p in pats], dtype=np.int64)[ip]
        for i, cg in zip(sel.tolist(), _cigars(ops, op_offsets, m + got[3], got[1] >= 0)):
            cigar[i] = cg
    with seqset._lock:
        pats = _bind_common(seqset._bind_many, subsequences)
        if pats is not None:
            align(np.arange(k), pats, lims, pidx)
        else:  # pattern by pattern, each bound (reducing the set to its own alphabet) right before its items
            for p in np.unique(pidx).tolist():
                sel = np.flatnonzero(pidx == p)
                align(sel, seqset._bind_many([subsequences[p]]), [lims[p]], np.zeros(sel.size, dtype=np.int64))
    return tuple(cols), cigar
