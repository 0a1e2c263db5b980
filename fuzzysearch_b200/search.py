"""The four search classes -- the reference's plugin seam (SURVEY.md section 8b).

``fuzzysearch.choose_search_class`` (__init__.py:60-83) picks one of ExactSearch /
SubstitutionsOnlySearch / LevenshteinSearch / GenericSearch, each a ``FuzzySearchBase`` with
``search(subsequence, sequence, search_params)`` and ``consolidate_matches(matches)``
(common.py:192-209).  Here each ``search`` is ONE call into libfuzzb200.so (sm_90a kernels);
there is no CPU implementation behind them.
"""
import threading
from collections.abc import Sequence

import numpy as np

from . import _native
from .common import FuzzySearchBase, Match, consolidate_overlapping_matches

try:  # optional, exactly like the reference (search_exact.py:14-19): Bio.Seq.Seq sequences are text
    from Bio.Seq import Seq as _BioSeq
except ImportError:
    _BioSeq = None


def _text(seq):
    """Bio.Seq.Seq -> its str (the reference walks a Seq with Seq.find / item access, i.e. as text); anything
    else unchanged.  ``Match.matched`` is still sliced from the ORIGINAL object."""
    if _BioSeq is not None and isinstance(seq, _BioSeq):
        return str(seq)
    return seq


__all__ = ["DeviceSequence", "ExactSearch", "SubstitutionsOnlySearch", "LevenshteinSearch",
           "GenericSearch", "RawMatches", "search_exact", "nearest_distance", "find_nearest_matches",
           "nearest_distance_batch", "find_nearest_matches_batch", "align_matches"]


class DeviceSequence(object):
    """A haystack kept resident in HBM so that several searches reuse one upload.

    ``find_near_matches(pattern, DeviceSequence(data), ...)`` behaves like
    ``find_near_matches(pattern, data, ...)``.  Byte-like data and latin-1 encodable ``str`` are uploaded
    once; a general-Unicode ``str`` (or a list / tuple of hashable items) is reduced to bytes relative to the
    PATTERN's alphabet (see ``_reduce``), so it is uploaded again whenever a search brings a pattern with a
    different set of symbols."""

    def __init__(self, data=None, device=0, _haystack=None, _host=None):
        # held across bind (re-reduction to a new pattern alphabet) + search + copy-out of the consolidated list:
        # threads sharing one resident sequence take turns, like callers of the reference under the GIL
        self._lock = threading.RLock()
        self._wide = None        # the original str / list / tuple when the byte form depends on the pattern
        self._alphabet = None    # ... and the pattern alphabet the resident bytes were reduced with
        self._is_str = False
        self._kind = "bytes"
        self._orig = None        # a Bio.Seq.Seq: `matched` is sliced from it
        if _haystack is not None:
            self.haystack, self._host = _haystack, _host
            return
        if _text(data) is not data:
            self._orig, data = data, _text(data)
        self._kind = _kind(data)
        self._is_str = self._kind == "str"
        host = _narrow(data, self._kind)
        if host is not None:
            self._host = host
            self.haystack = _native.Haystack.from_host(host, device=device)
        else:
            self._host = None
            self._wide = data
            self.haystack = _native.Haystack.alloc(max(len(data), 1), device=device)

    def __len__(self):
        if self._orig is not None:
            return len(self._orig)
        return len(self._wide) if self._wide is not None else len(self.haystack)

    def _bind(self, subsequence):
        """-> the pattern as bytes in this sequence's byte alphabet (re-reducing the sequence if needed)."""
        return self._bind_many([subsequence])[0]

    def _bind_many(self, subsequences):
        subsequences = [_text(p) for p in subsequences]
        kinds = set(_kind(p) for p in subsequences)
        if kinds != {self._kind}:
            raise TypeError("subsequence and sequence must both be str or both be byte-like")
        if self._wide is None:
            pats = [_narrow(p, self._kind) for p in subsequences]
            if all(p is not None for p in pats):
                return pats
            # a pattern with symbols outside latin-1 over a latin-1 sequence: those symbols match nothing,
            # but the search still has to run with them in place -- reduce both sides
            self._wide = self.slice(0, len(self))
        alphabet = _make_alphabet(subsequences, self._kind)
        if alphabet != self._alphabet:
            _upload_reduced(self.haystack, self._wide, self._kind, alphabet)
            self._alphabet = alphabet
        return [_rename(p, self._kind, alphabet) for p in subsequences]

    def slice(self, start, end):
        if self._orig is not None:
            return self._orig[start:end]
        if self._wide is not None:
            return self._wide[start:end]
        if self._host is not None:
            b = bytes(memoryview(self._host)[start:end])
        else:
            b = self.haystack.read(start, end - start)
        return b.decode("latin-1") if self._is_str else b

    def close(self):
        self.haystack.close()


def _kind(seq):
    """'str' | 'items' (list / tuple of hashable items) | 'bytes' (anything byte-like)"""
    if isinstance(seq, str):
        return "str"
    if isinstance(seq, (list, tuple)):
        return "items"
    return "bytes"


def _narrow(seq, kind):
    """-> uint8 view when `seq` has single-byte symbols of its own (byte-like: zero-copy; latin-1 encodable
    str: encoded), else None."""
    if kind == "str":
        try:
            return np.frombuffer(seq.encode("latin-1"), dtype=np.uint8)
        except UnicodeEncodeError:
            return None
    if kind == "items":
        return None
    return _native.as_u8(seq)


def _coerce(seq):
    """-> (uint8 view, is_str) for sequences with single-byte symbols."""
    kind = _kind(seq)
    a = _narrow(seq, kind)
    if a is None:
        raise TypeError("a sequence of single-byte symbols is required here (got %s)" % type(seq).__name__)
    return a, kind == "str"


class AlphabetTooLarge(_native.UnsupportedError):
    pass


def _bind_common(bind, *args):
    """-> bind(*args), or None when the patterns it binds have no common byte alphabet (wide symbols and more than 255
    distinct ones over all of them): the caller then takes the patterns one by one, each reducing the sequence to its
    own alphabet."""
    try:
        return bind(*args)
    except AlphabetTooLarge:
        return None


def _make_alphabet(subsequences, kind):
    """The reduction every algorithm on the path is invariant under (they only ever compare a pattern symbol
    with a sequence symbol -- levenshtein_ngram.py:49,113, levenshtein.py:83, generic_search.py:86,
    substitutions_only.py:93-99, search_exact.py:45-56): pattern symbol -> 1 + its rank among the distinct
    symbols of the pattern(s), any other sequence symbol -> 0.

    str: the sorted code points (the device reduces the sequence side, k_reduce_symbols);
    items: {item: byte} (Python objects can only be numbered by the interpreter)."""
    if kind == "str":
        alphabet = sorted(set(ord(c) for p in subsequences for c in p))
        if len(alphabet) > _native.FZB_MAX_PATTERN:
            raise AlphabetTooLarge("more than %d distinct pattern symbols" % _native.FZB_MAX_PATTERN)
        return alphabet
    ids = {}
    for p in subsequences:
        for item in p:
            if item not in ids:
                if len(ids) == _native.FZB_MAX_PATTERN:
                    raise AlphabetTooLarge("more than %d distinct pattern symbols" % _native.FZB_MAX_PATTERN)
                ids[item] = len(ids) + 1
    return ids


def _rename(subsequence, kind, alphabet):
    if kind == "str":
        rank = {c: i + 1 for i, c in enumerate(alphabet)}
        return np.fromiter((rank[ord(c)] for c in subsequence), dtype=np.uint8, count=len(subsequence))
    return np.fromiter((alphabet[x] for x in subsequence), dtype=np.uint8, count=len(subsequence))


def _code_units(text):
    """str -> its code units as a numpy array: UCS-2 (uint16) when every character is in the BMP, else
    UTF-32 (uint32).  Lone surrogates are symbols like any other ('surrogatepass')."""
    if not text or max(text) < "\U00010000":
        return np.frombuffer(text.encode("utf-16-le", "surrogatepass"), dtype=np.uint16)
    return np.frombuffer(text.encode("utf-32-le", "surrogatepass"), dtype=np.uint32)


def _upload_reduced(hay, sequence, kind, alphabet):
    if kind == "str":
        hay.upload_symbols(_code_units(sequence), alphabet)
    else:
        get = alphabet.get
        try:
            hay.upload(np.fromiter((get(x, 0) for x in sequence), dtype=np.uint8, count=len(sequence)))
        except TypeError:
            raise TypeError("sequence items must be hashable")


class RawMatches(Sequence):
    """The raw match stream of one search, materialised LAZILY: ``find_near_matches`` only needs the
    consolidated list (``.final``, built from the device-side consolidation), so the raw ``Match``
    objects -- one Python object and one slice per raw record -- are only built if somebody iterates,
    indexes or compares this object (the search-class ``search()`` contract of the reference,
    common.py:192-197, is "an iterable of Match")."""

    def __init__(self, result, slicer, consolidated):
        self._result = result
        self._slicer = slicer
        self._list = None
        self.stats = result.stats()
        self.final = _to_matches(result.arrays(_native.FINAL), slicer) if consolidated else None
        self._n = result.count(_native.RAW)

    def materialize(self):
        if self._list is None:
            self._list = _to_matches(self._result.arrays(_native.RAW), self._slicer)
            self._result.close()
            self._result = None
        return self._list

    def __len__(self):
        return self._n

    def __iter__(self):
        return iter(self.materialize())

    def __getitem__(self, i):
        return self.materialize()[i]

    def __eq__(self, other):
        if isinstance(other, RawMatches):
            other = other.materialize()
        return self.materialize() == other

    def __ne__(self, other):
        return not self.__eq__(other)

    __hash__ = None

    def __repr__(self):
        return repr(self.materialize())

    def __del__(self):
        if getattr(self, "_result", None) is not None:
            self._result.close()


def _prepare(subsequence, sequence):
    """-> (pattern u8, haystack handle, slicer)"""
    pats, hay, slicer = _prepare_many([subsequence], sequence)
    return pats[0], hay, slicer


def _prepare_many(subsequences, sequence):
    """-> (patterns as u8 arrays, haystack handle holding the sequence, slicer)"""
    if isinstance(sequence, DeviceSequence):
        return sequence._bind_many(subsequences), sequence.haystack, sequence.slice
    original, sequence = sequence, _text(sequence)
    subsequences = [_text(p) for p in subsequences]
    kind = _kind(sequence)
    if any(_kind(p) != kind for p in subsequences):
        raise TypeError("subsequence and sequence must both be str or both be byte-like")
    pats = [_narrow(p, kind) for p in subsequences]
    host = _narrow(sequence, kind) if all(p is not None for p in pats) else None
    if host is not None:
        hay = _workspace(host.size)
        hay.upload(host)
    else:  # wide symbols on either side: reduce both to the patterns' alphabet
        alphabet = _make_alphabet(subsequences, kind)
        pats = [_rename(p, kind, alphabet) for p in subsequences]
        hay = _workspace(len(sequence))
        _upload_reduced(hay, sequence, kind, alphabet)
    return pats, hay, _slicer(original, kind, host)


def _slicer(original, kind, u8=None):
    """Match.matched as find_near_matches(pattern, original) slices it: a slice of the original object, as bytes for a
    byte-like object other than bytes / bytearray (u8: its uint8 view, when the caller already has it)."""
    if kind != "bytes" or isinstance(original, (bytes, bytearray)):
        return lambda s, e: original[s:e]
    mv = memoryview(_native.as_u8(original) if u8 is None else u8)
    return lambda s, e: bytes(mv[s:e])


_WORKSPACE = {}
# One lock per process around upload + search + copy-out of the SHARED workspace: ctypes drops the GIL
# during the native calls, so without it two threads calling find_near_matches() would overwrite each
# other's haystack mid-search.  (The reference is serialised by the GIL.)  A DeviceSequence has its own lock
# (and the library serialises the calls on one handle), so searches of different resident sequences overlap.
_WORKSPACE_LOCK = threading.RLock()


def _lock_for(sequence):
    return sequence._lock if isinstance(sequence, DeviceSequence) else _WORKSPACE_LOCK


def _workspace(nbytes, device=0):
    """A cached device buffer for plain (host) sequences: like the reference's reusable chunk buffer
    (__init__.py:141-145), a search then costs one H2D copy instead of allocations."""
    ws = _WORKSPACE.get(device)
    if ws is None or ws[1] < nbytes:
        if ws is not None:
            ws[0].close()
        cap = max(nbytes + nbytes // 8, 1 << 20)
        ws = (_native.Haystack.alloc(cap, device=device), cap)
        _WORKSPACE[device] = ws
    return ws[0]


def release_workspace():
    for ws in _WORKSPACE.values():
        ws[0].close()
    _WORKSPACE.clear()
    _native.lib().fzb_release_workspace()


def _matches(starts, ends, dists, slicer):
    """(start, end, dist) lists of ints -> the Match list, `matched` cut by slicer."""
    return [Match(a, b, c, matched=slicer(a, b)) for a, b, c in zip(starts, ends, dists)]


def _to_matches(arrays, slicer):
    """The (start, end, dist) arrays of a list -> its Match list."""
    return _matches(*(x.tolist() for x in arrays), slicer)


def _check_pattern(cls, subsequence):
    """The empty-pattern refusal of cls.search (ExactSearch words it as search_exact does)."""
    if len(subsequence) == 0:
        raise ValueError("subsequence must not be empty" if cls is ExactSearch else "Given subsequence is empty!")


def _max_substitutions(search_params):
    """The limit SubstitutionsOnlySearch.search applies (substitutions_only.py:288-301)."""
    return min(x for x in (search_params.max_l_dist, search_params.max_substitutions) if x is not None)


def _list_of(cls):
    """Which list of a search of class cls find_near_matches returns: ExactSearch does not consolidate
    (search_exact.py:80-89), its list is the RAW stream of the k == 0 route; the others the FINAL list (the Hamming
    FINAL list equals RAW)."""
    return _native.RAW if cls is ExactSearch else _native.FINAL


def _search_one(cls, hay, pat, search_params):
    """One pattern searched on the handle `hay` as cls.search searches it -> (Result, the list to read)."""
    if cls is ExactSearch:
        res = hay.search_exact(pat)
    elif cls is SubstitutionsOnlySearch:
        res = hay.search_hamming(pat, _max_substitutions(search_params))
    elif cls is LevenshteinSearch:
        res = hay.search_levenshtein(pat, search_params.max_l_dist)
    else:
        res = hay.search_generic(pat, *search_params.unpacked)
    return res, _list_of(cls)


def _search_class(cls, subsequence, sequence, search_params, consolidated):
    """cls.search: the pattern checked, then searched as _search_one searches it -> RawMatches."""
    _check_pattern(cls, subsequence)
    return _run(subsequence, sequence, lambda h, p: _search_one(cls, h, p, search_params)[0], consolidated)


def _run(subsequence, sequence, call, consolidated):
    with _lock_for(sequence):
        pat, hay, slicer = _prepare(subsequence, sequence)
        res = call(hay, pat)
        try:
            return RawMatches(res, slicer, consolidated)
        except BaseException:
            res.close()
            raise


def search_exact(subsequence, sequence, start_index=0, end_index=None):
    """fuzzysearch.search_exact.search_exact (search_exact.py:22-56): the start indexes of the (overlapping)
    occurrences of `subsequence` lying wholly inside ``sequence[start_index:end_index]``, ascending.

    Only the window travels to / is scanned on the device: a host sequence is sliced before the upload, a
    ``DeviceSequence`` is searched through a view of its resident buffer (fzb_search_exact_window)."""
    if len(subsequence) == 0:
        raise ValueError("subsequence must not be empty")
    sequence = _text(sequence)  # a Bio.Seq.Seq is searched as its text; the result is positions only
    n = len(sequence)
    if end_index is None:
        end_index = n
    start_index = max(0, min(start_index, n))               # clamp(...) search_exact.py:29-30
    end_index = max(start_index, min(end_index, n))
    if isinstance(sequence, DeviceSequence):
        with sequence._lock:
            pat = sequence._bind(subsequence)
            res = sequence.haystack.search_exact(pat, start=start_index, end=end_index)
            starts = res.arrays(_native.RAW)[0]  # positions are already those of the whole sequence
            res.close()
        return starts.tolist()
    else:
        if _kind(sequence) == "bytes" and not isinstance(sequence, (bytes, bytearray)):
            window = memoryview(_native.as_u8(sequence))[start_index:end_index]
        elif start_index == 0 and end_index == n:
            window = sequence
        else:
            window = sequence[start_index:end_index]
        with _WORKSPACE_LOCK:
            pat, hay, _ = _prepare(subsequence, window)
            res = hay.search_exact(pat)
            starts = res.arrays(_native.RAW)[0]
            res.close()
        return (starts + start_index).tolist() if start_index else starts.tolist()


class ExactSearch(FuzzySearchBase):
    """search_exact.py:80-89."""

    @classmethod
    def search(cls, subsequence, sequence, search_params=None):
        return _search_class(ExactSearch, subsequence, sequence, search_params, False)

    @classmethod
    def extra_items_for_chunked_search(cls, subsequence, search_params):
        return 0


class SubstitutionsOnlySearch(FuzzySearchBase):
    """substitutions_only.py:288-301."""

    @classmethod
    def search(cls, subsequence, sequence, search_params):
        return _search_class(SubstitutionsOnlySearch, subsequence, sequence, search_params, False)

    @classmethod
    def extra_items_for_chunked_search(cls, subsequence, search_params):
        return 0


class LevenshteinSearch(FuzzySearchBase):
    """levenshtein.py:151-164."""

    @classmethod
    def search(cls, subsequence, sequence, search_params):
        return _search_class(LevenshteinSearch, subsequence, sequence, search_params, True)

    @classmethod
    def consolidate_matches(cls, matches):
        return consolidate_overlapping_matches(matches)

    @classmethod
    def extra_items_for_chunked_search(cls, subsequence, search_params):
        return search_params.max_l_dist


class GenericSearch(FuzzySearchBase):
    """generic_search.py:256-273."""

    @classmethod
    def search(cls, subsequence, sequence, search_params):
        return _search_class(GenericSearch, subsequence, sequence, search_params, True)

    @classmethod
    def consolidate_matches(cls, matches):
        return consolidate_overlapping_matches(matches)

    @classmethod
    def extra_items_for_chunked_search(cls, subsequence, search_params):
        return max(x for x in [search_params.max_l_dist, search_params.max_insertions] if x is not None)


def _nearest_flags(substitutions_only, anchor=None):
    """The flags of the nearest_* calls; ValueError for an anchor other than None, 'start' or 'end'."""
    flags = _native.F_SUBSTITUTIONS_ONLY if substitutions_only else 0
    if anchor is None:
        return flags
    if isinstance(anchor, str) and anchor == "start":
        return flags | _native.F_ANCHOR_START
    if isinstance(anchor, str) and anchor == "end":
        return flags | _native.F_ANCHOR_END
    raise ValueError("anchor must be None, 'start' or 'end', not %r" % (anchor,))


def _nearest_params(d, substitutions_only):
    """The limits at which find_near_matches lists the matches at the nearest distance d -> (params, search class)."""
    from . import choose_search_class
    from .common import LevenshteinSearchParams
    params = (LevenshteinSearchParams(d, 0, 0, None) if substitutions_only else
              LevenshteinSearchParams(None, None, None, d))
    return params, choose_search_class(params)


def nearest_distance(subsequence, sequence, *, substitutions_only=False):
    """The smallest Levenshtein distance of `subsequence` to any substring of `sequence` (at most
    ``len(subsequence)``: the empty substring) -- the smallest ``max_l_dist`` at which ``find_near_matches`` finds
    anything.  One scan of the sequence, whatever the answer (fzb_nearest_distance, DESIGN.md section 5.14).
    `sequence` is anything find_near_matches takes.

    With ``substitutions_only=True``: the smallest number of substitutions of any window of ``len(subsequence)``
    symbols -- the smallest k at which ``find_near_matches(..., max_substitutions=k, max_insertions=0,
    max_deletions=0)`` finds anything -- or None when the sequence is shorter than the pattern (DESIGN.md section
    5.16)."""
    if len(subsequence) == 0:
        raise ValueError("Given subsequence is empty!")
    with _lock_for(sequence):
        pat, hay, _ = _prepare(subsequence, sequence)
        d = hay.nearest_distance(pat, _nearest_flags(substitutions_only))[0]
        return None if d == _native.NO_DIST else d


def find_nearest_matches(subsequence, sequence, max_l_dist=None, *, substitutions_only=False):
    """Where does `subsequence` fit best?  -> exactly ``find_near_matches(subsequence, sequence, max_l_dist=d)`` with
    d = ``nearest_distance(subsequence, sequence)``, without guessing d: one scan finds it, then the ordinary search
    runs once, at d, on the same upload.  With `max_l_dist` given the list is empty when d is larger (the cap bounds
    the cost of the search; the search itself still runs at d, not at the cap).

    With ``substitutions_only=True``: exactly ``find_near_matches(subsequence, sequence, max_substitutions=d,
    max_insertions=0, max_deletions=0)`` with d = ``nearest_distance(..., substitutions_only=True)``, and [] when
    the sequence is shorter than the pattern.  Every window at d is listed, so a d close to ``len(subsequence)``
    lists almost every window; the cap avoids that."""
    if len(subsequence) == 0:
        raise ValueError("Given subsequence is empty!")
    if max_l_dist is not None and (not isinstance(max_l_dist, int) or max_l_dist < 0):
        raise ValueError("max_l_dist must be a non-negative integer or None")
    with _lock_for(sequence):
        pat, hay, slicer = _prepare(subsequence, sequence)
        d = hay.nearest_distance(pat, _nearest_flags(substitutions_only))[0]
        if d == _native.NO_DIST or (max_l_dist is not None and d > max_l_dist):
            return []
        params, cls = _nearest_params(d, substitutions_only)
        res, which = _search_one(cls, hay, pat, params)
        try:
            return _to_matches(res.arrays(which), slicer)
        finally:
            res.close()


def _nearest_batch(subsequences, sequence, flags):
    """-> (dist int32, first end int64) arrays, one entry per pattern, -1 / -1 without a value.  The caller holds
    the sequence's lock."""
    bound = _bind_common(_prepare_many, subsequences, sequence)
    if bound is not None:
        dist, end, _ = bound[1].nearest_distance_batch(bound[0], flags)
        return dist, end
    rows = []
    for p in subsequences:
        pat, hay, _ = _prepare(p, sequence)
        d, _, e, _ = hay.nearest_distance(pat, flags)
        rows.append((-1, -1) if d == _native.NO_DIST else (d, e))
    return np.array([d for d, _ in rows], dtype=np.int32), np.array([e for _, e in rows], dtype=np.int64)


def nearest_distance_batch(subsequences, sequence, *, substitutions_only=False):
    """Many patterns over one sequence, without a distance limit: -> NearestDistances with one entry per pattern,
    ``dist[i] == nearest_distance(subsequences[i], sequence)`` and ``end[i]`` the first end position of a substring at
    that distance.  The patterns of up to 64 symbols share scans of the sequence, 32 at a time
    (fzb_nearest_distance_batch, DESIGN.md section 5.15).  `sequence` is anything find_near_matches takes.  With
    ``substitutions_only=True`` the distances are ``nearest_distance(..., substitutions_only=True)``, and a pattern
    longer than the sequence gets -1 / -1."""
    from .sequence_set import NearestDistances
    subsequences = list(subsequences)
    if any(len(p) == 0 for p in subsequences):
        raise ValueError("Given subsequence is empty!")
    if not subsequences:
        return NearestDistances(np.zeros(0, np.int32), np.zeros(0, np.int64))
    with _lock_for(sequence):
        return NearestDistances(*_nearest_batch(subsequences, sequence, _nearest_flags(substitutions_only)))


def find_nearest_matches_batch(subsequences, sequence, max_l_dist=None, *, substitutions_only=False):
    """Where does each pattern fit best?  -> exactly ``find_near_matches_batch(subsequences, sequence,
    max_l_dist=[d_0, d_1, ...])`` with d_i = ``nearest_distance(subsequences[i], sequence)``, found by one batch of
    shared scans and searched on the same upload.  `max_l_dist` (None, one int, or one value per pattern) caps d_i:
    a pattern whose d_i is larger gets ``[]`` and is not searched.  With ``substitutions_only=True``: exactly
    ``find_near_matches_batch(..., max_substitutions=[d_0, d_1, ...], max_insertions=0, max_deletions=0)`` with the
    substitutions-only d_i, and ``[]`` for a pattern longer than the sequence."""
    from . import _search_batch
    subsequences = list(subsequences)
    n = len(subsequences)
    caps = max_l_dist if isinstance(max_l_dist, (list, tuple)) else [max_l_dist] * n
    if len(caps) != n:
        raise ValueError("one max_l_dist per subsequence expected")
    if any(c is not None and (not isinstance(c, int) or c < 0) for c in caps):
        raise ValueError("max_l_dist must be a non-negative integer or None")
    if any(len(p) == 0 for p in subsequences):
        raise ValueError("Given subsequence is empty!")
    if not subsequences:
        return []
    with _lock_for(sequence):
        bound = _bind_common(_prepare_many, subsequences, sequence)
        if bound is None:
            return [find_nearest_matches(p, sequence, c, substitutions_only=substitutions_only)
                    for p, c in zip(subsequences, caps)]
        pats, hay, slicer = bound
        dist, _, _ = hay.nearest_distance_batch(pats, _nearest_flags(substitutions_only))
        todo = [i for i in range(n) if dist[i] >= 0 and (caps[i] is None or dist[i] <= caps[i])]
        found = [_nearest_params(int(dist[i]), substitutions_only) for i in todo]
        lists = _search_batch(hay, [pats[i] for i in todo], [p for p, _ in found], [c for _, c in found], 0)
    out = [[] for _ in range(n)]
    for i, arrays in zip(todo, lists):
        out[i] = _to_matches(arrays, slicer)
    return out


_BIG = 1 << 29  # an absent limit, as the batches pass it to the library


def _normalised_limits(search_params):
    """-> (max_subs, max_ins, max_dels, max_l) as the library takes them: None becomes a limit that never binds."""
    return tuple(_BIG if x is None else min(x, _BIG) for x in search_params.unpacked)


def _cigars(ops, op_offsets, n_ops, valid):
    """The op bytes of every item (fzb_align) -> one extended CIGAR string per item, '' where `valid` is false.  The
    runs are found and counted in numpy: a run starts at each item's first op and wherever the op changes."""
    out = [""] * len(valid)
    idx = np.flatnonzero(valid)
    if idx.size == 0:
        return out
    lens = np.asarray(n_ops, dtype=np.int64)[idx]
    first = np.cumsum(lens) - lens  # each item's first op in the gathered array
    total = int(lens.sum())
    item_of = np.repeat(np.arange(idx.size), lens)
    flat = ops[np.asarray(op_offsets, dtype=np.int64)[idx][item_of] + (np.arange(total) - first[item_of])]
    brk = np.empty(total, dtype=bool)
    brk[0] = True
    brk[1:] = flat[1:] != flat[:-1]
    brk[first] = True
    runs = np.flatnonzero(brk)
    lengths = np.diff(np.append(runs, total))
    text = np.strings.add(lengths.astype(np.str_), flat[runs].view("S1").astype(np.str_))
    ends = np.searchsorted(runs, first[1:]) - 1  # the last run of every item but the last one
    text[ends] = np.strings.add(text[ends], "\n")
    for i, c in zip(idx.tolist(), "".join(text.tolist()).split("\n")):
        out[i] = c
    return out


def align_matches(subsequence, sequence, matches, max_substitutions=None, max_insertions=None, max_deletions=None,
                  max_l_dist=None):
    """The edit operations of matches: -> one extended CIGAR string per Match, in sequence order ('=' equal, 'X'
    substituted, 'I' a sequence symbol the pattern lacks, 'D' a pattern symbol the sequence lacks), e.g.
    ``'5=1X3=1I10='``.  Pass the limits of the search that produced `matches`; they select the cost model as
    find_near_matches selects its search (fzb_align, DESIGN.md section 5.17).  `sequence` is anything
    find_near_matches takes.  Each match is aligned on the device, one warp per match; the alignment is the cheapest
    one of the pattern against ``sequence[start:end]``, the canonical one among equals.  Its cost is at most
    ``Match.dist``: exactly it for the exact and substitutions-only searches, ``lev(subsequence, matched)`` for
    Levenshtein, which can be below ``Match.dist``.  A match with no alignment within its dist and the limits (a
    wrong pattern, sequence or limit) raises ValueError."""
    from .common import LevenshteinSearchParams
    search_params = LevenshteinSearchParams(max_substitutions, max_insertions, max_deletions, max_l_dist)
    if len(subsequence) == 0:
        raise ValueError("Given subsequence is empty!")
    matches = list(matches)
    if not matches:
        return []
    s = np.fromiter((x.start for x in matches), dtype=np.int64, count=len(matches))
    e = np.fromiter((x.end for x in matches), dtype=np.int64, count=len(matches))
    d = np.fromiter((x.dist for x in matches), dtype=np.int32, count=len(matches))
    if (s < 0).any() or (d < 0).any():
        raise ValueError("matches need non-negative starts and dists")
    lims = _normalised_limits(search_params)
    with _lock_for(sequence):
        pat, hay, _ = _prepare(subsequence, sequence)
        (_, cost, _, ins, _), ops, op_offsets, _ = hay.align([pat], *[[x] for x in lims], np.zeros(len(matches)), s,
                                                             e, d)
    bad = np.flatnonzero(cost < 0)
    if bad.size:
        raise ValueError("no alignment of the subsequence within the dist and limits of %r" % (matches[int(bad[0])],))
    return _cigars(ops, op_offsets, len(pat) + ins, cost >= 0)
