"""The multi-rank reduction k_push -> k_merge (csrc/p2p_kernels.cuh, DESIGN section 6) at its seam, slot and ownership
limits, on in-process worlds of 2-8 shards on one device.

Every case compares the merge with a restatement of the global consolidation written from its definition
(consolidate_overlapping_matches, common.py:145-189), not from the kernel: every rank's own group rows
(start, end, dist, hull_start, hull_end) of the same search without F_GLOBAL, ordered by (hull_start, rank, index); a
row heads a group iff it is the first or its hull starts at or after the largest hull end before it; the winner of a
group is its smallest (dist, -length, start).  The restated group and non-head counts are checked against the merge's
own (debug_counters()[17] and [22], status [16]), and every case asserts from the restated rows that it reaches the
branch of p2p_kernels.cuh it names."""
import contextlib

import numpy as np
import pytest

import oracle
from fuzzysearch_b200 import _native as F
from fuzzysearch_b200.sharding import ALIGN, init_local_world, search_all, shard_bounds
from parity import tup

pytestmark = pytest.mark.gpu

CAP = 4096           # group rows of one peer slot (api.cu: p2p_cap)
POST_MAX = 16384     # raw records k_post consolidates (post_kernels.cuh: kPostMax)
THREADS = 1024       # k_merge's CTA: phase 1 strides over a run, phase 3 over W runs by this
MS_OK = 1


# ---- the restatement ---------------------------------------------------------------------------------------------
def restate(runs, consolidated=True):
    """runs[r]: rank r's group rows (s, e, d, hull_s, hull_e) -> dict with the global final triples, the group count,
    the non-head rows (rank, index, hull_s) and the ordered rows."""
    rows = sorted((int(hs), r, i, int(s), int(e), int(d), int(he))
                  for r, run in enumerate(runs) for i, (s, e, d, hs, he) in enumerate(np.asarray(run).reshape(-1, 5)))
    if not consolidated:  # exact, Hamming: the global list is the sorted union
        return {"final": sorted((s, e, d) for _, _, _, s, e, d, _ in rows), "groups": len(rows), "nonheads": [],
                "rows": rows, "group_ranks": [{r} for _, r, *_ in rows]}
    groups, ranks, nonheads, reach = [], [], [], None
    for hs, r, i, s, e, d, he in rows:
        if groups and hs < reach:  # an earlier hull reaches past this hull's start: same group
            groups[-1].append((s, e, d))
            ranks[-1].add(r)
            nonheads.append((r, i, hs))
            reach = max(reach, he)
        else:
            groups.append([(s, e, d)])
            ranks.append({r})
            reach = he
    final = sorted(min(g, key=lambda t: (t[2], -(t[1] - t[0]), t[0])) for g in groups)
    return {"final": final, "groups": len(groups), "nonheads": nonheads, "rows": rows, "group_ranks": ranks}


def equal_hull_starts(rows):
    """hull starts that rows of two different ranks share"""
    ranks = {}
    for hs, r, *_ in rows:
        ranks.setdefault(hs, set()).add(r)
    return sorted(hs for hs, rs in ranks.items() if len(rs) > 1)


def interleaved(runs):
    """(q, r) pairs where a row of rank q has its hull start strictly inside rank r's range of hull starts: k_merge
    binary-searches run r for that row"""
    out = set()
    for q, a in enumerate(runs):
        for r, b in enumerate(runs):
            if q != r and len(a) and len(b):
                if any(b[0][3] < hs < b[-1][3] for hs in a[:, 3]):
                    out.add((q, r))
    return out


# ---- worlds ------------------------------------------------------------------------------------------------------
def seams_of(n, world, halo):
    return [shard_bounds(n, world, r, halo)[2:] for r in range(world)]


@contextlib.contextmanager
def local_world(hay, bounds, halo, device):
    """One handle per owned range [lo, hi) of `bounds` (any partition of [0, n) into 16-aligned ranges, empty ones
    included), each loading its range plus `halo` on both sides."""
    n = len(hay)
    shards = []
    try:
        for lo, hi in bounds:
            blo = max(0, lo - halo) // ALIGN * ALIGN
            bhi = max(min(n, hi + halo), blo + 1)
            shards.append(F.Haystack.from_host(hay[blo:bhi], device=device, buf_lo=blo, global_len=n, own_lo=lo,
                                               own_hi=hi))
        init_local_world(shards)
        yield shards
    finally:
        for h in shards:
            h.close()


def check_merge(shards, hay, search, exp, consolidated=True, device=0):
    """search(h, flags) -> Result.  Every rank's F_GLOBAL list against the restatement of the ranks' own rows and
    against `exp` (the oracle on the whole sequence); the merge's status, group and non-head counts; the ranks' raw
    streams against the single-device raw stream.  -> the restatement, with each rank's raw count added."""
    runs, raws, raw_counts = [], [], []
    for h in shards:
        res = search(h, 0)
        runs.append(res.group_rows())
        raws += res.triples(F.RAW)
        raw_counts.append(h.debug_counters()[0])
    want = restate(runs, consolidated)
    assert want["final"] == exp
    got = search_all(shards, lambda h: (search(h, F.F_GLOBAL).triples(F.FINAL), h.debug_counters()))
    for r, (fin, dbg) in enumerate(got):
        assert fin == exp, r
        assert dbg[16] == MS_OK, (r, dbg[16])
        assert dbg[17] == want["groups"], (r, dbg[17], want["groups"])
        assert dbg[22] == len(want["nonheads"]), (r, dbg[22], len(want["nonheads"]))
    whole = F.Haystack.from_host(hay, device=device)
    try:
        assert sorted(raws) == sorted(search(whole, 0).triples(F.RAW))
    finally:
        whole.close()
    want["runs"] = runs
    want["raw_counts"] = raw_counts
    return want


def lev(pat, k, extra=0):
    return lambda h, flags: h.search_levenshtein(pat, k, flags | extra)


def lev_oracle(pat, hay, k):
    return oracle.find_near_matches(pat, hay, max_l_dist=k)


def guarded(call):
    """search_all body that hands back the exception of a rank instead of raising it"""
    def run(h):
        try:
            return call(h)
        except Exception as e:  # noqa: BLE001 -- compared by the caller, rank by rank
            return e
    return run


def digits(n, seed):
    """a text of digits: no byte of the letter patterns below, so the plants are the only matches"""
    return np.random.default_rng(seed).integers(48, 58, size=n, dtype=np.uint8)


def put(hay, pos, b):
    hay[pos:pos + len(b)] = np.frombuffer(bytes(b), dtype=np.uint8)


PERIODIC = b"abcdefghij" * 2  # period 10: copies 10 apart overlap, so groups of two ranks meet near a seam
TOUCHING = b"klmnopqrstuvwxyzABCD"  # no period: two copies back to back are two groups that touch


def seam_run(subs=(), ins=None):
    """30 bytes of PERIODIC's period with substitutions (index, byte) and one inserted 'Z' (at `ins`)"""
    run = bytearray(b"abcdefghij" * 3)
    for i, c in subs:
        run[i] = c
    if ins is not None:
        run[ins:ins] = b"Z"
    return bytes(run)


# Seam constructions for m = 20, k = 2 (offset of the run from the seam, run bytes) and what they make k_merge meet
# at that seam (found by restating the per-rank groups of the oracle's raw stream, tests/test_emu_world_merge.py).
SEAM_CASES = {
    # a group of rank q - 1 and one of rank q with the SAME hull start: phase 1 orders them by rank (`low && v == hs`)
    "equal_hs_higher_longer": (-12, seam_run([(10, ord("Y"))])),
    "equal_hs_lower_longer": (-12, seam_run([(18, ord("X")), (22, ord("Y"))])),
    # one global group, the two runs' winners tie in distance: the longer wins / at equal length the earlier start
    "tie_length": (-23, seam_run([(21, ord("Y"))], ins=1)),
    "tie_start": (-22, seam_run()),
}


def test_equal_hull_starts_and_winner_ties(cuda_device, small=False):
    """Case 1.  World 5 (4 seams), one construction per seam; then every construction at every seam of a world of 3."""
    m, k, n = 20, 2, 1 << 14
    for world in (5, 3):
        bounds = seams_of(n, world, m + k)
        names = list(SEAM_CASES)
        for shift in range(len(names) if world == 3 and not small else 1):
            hay = digits(n, 11 + shift)
            placed = {}
            for r in range(1, world):
                name = names[(r - 1 + shift) % len(names)]
                off, run = SEAM_CASES[name]
                put(hay, bounds[r][0] + off, run)
                placed[r] = name
            with local_world(hay, bounds, m + k, cuda_device) as shards:
                got = check_merge(shards, hay, lev(PERIODIC, k), lev_oracle(PERIODIC, hay, k), device=cuda_device)
            runs = got["runs"]
            assert got["groups"] == world - 1 and len(got["nonheads"]) == world - 1
            for q, name in placed.items():  # the branch each seam claims, from the ranks' own rows
                lower, higher = runs[q - 1][-1], runs[q][0]
                if name.startswith("equal_hs"):
                    assert lower[3] == higher[3], (name, lower, higher)
                    longer = lower if name.endswith("lower_longer") else higher
                    shorter = higher if longer is lower else lower
                    assert longer[4] > shorter[4], (name, lower, higher)
                elif name == "tie_length":
                    assert lower[2] == higher[2] and lower[1] - lower[0] != higher[1] - higher[0], (lower, higher)
                else:
                    assert lower[2] == higher[2] and lower[1] - lower[0] == higher[1] - higher[0], (lower, higher)
                    assert lower[0] != higher[0], (lower, higher)


def test_touching_and_interleaved_hulls(cuda_device, small=False):
    """Case 2.  At seam 1 a copy of TOUCHING ends exactly where a copy anchored on the next rank starts: two groups
    (`he > hs` is strict).  At seam 2 (as in test_gpu_global.test_seam_rows_interleave_between_runs) a row of rank 2
    starts between two rows of rank 1: the binary search places it, its head test must read row nb - 1 of run 1, whose
    hull ends before it, and not run 1's last row, whose hull reaches past it; that last row is the one non-head."""
    m, k, n, world = 20, 2, 1 << 13, 3
    bounds = seams_of(n, world, m + k)
    hay = digits(n, 21)
    s1, s2 = bounds[1][0], bounds[2][0]
    put(hay, s1 - 20, TOUCHING)
    put(hay, s1, TOUCHING)
    put(hay, s2 - 300, PERIODIC)
    put(hay, s2 - 12, seam_run([(2, ord("X")), (8, ord("Y"))]))
    with local_world(hay, bounds, m + k, cuda_device) as shards:
        touch = check_merge(shards, hay, lev(TOUCHING, k), lev_oracle(TOUCHING, hay, k), device=cuda_device)
        got = check_merge(shards, hay, lev(PERIODIC, k), lev_oracle(PERIODIC, hay, k), device=cuda_device)
    runs = touch["runs"]
    assert runs[0][-1][4] == runs[1][0][3] == s1 and touch["groups"] == 2 and not touch["nonheads"]
    runs = got["runs"]
    assert (2, 1) in interleaved(runs)
    r2 = runs[2][0]
    nb = int(np.searchsorted(runs[1][:, 3], r2[3], side="right"))
    assert 0 < nb < len(runs[1]) and runs[1][nb - 1][4] <= r2[3] < runs[1][-1][4]
    assert [(r, i) for r, i, _ in got["nonheads"]] == [(1, len(runs[1]) - 1)]


def test_groups_chain_over_every_rank(cuda_device, small=False):
    """Case 3.  World 8, ranks 1-6 own 16 or 32 bytes each, on a periodic stretch of text: one global group takes a row
    from every rank, so every seam's rows are non-heads behind a chain that crosses several seams."""
    m, k, n = 20, 2, 1024
    edges = [0, 400, 416, 448, 464, 496, 512, 544, n]
    bounds = list(zip(edges[:-1], edges[1:]))
    hay = digits(n, 31)
    put(hay, 300, b"abcdefghij" * 40)
    with local_world(hay, bounds, m + k, cuda_device) as shards:
        got = check_merge(shards, hay, lev(PERIODIC, k), lev_oracle(PERIODIC, hay, k), device=cuda_device)
    assert set(range(8)) in got["group_ranks"], got["group_ranks"]
    assert len(got["nonheads"]) >= 7


def test_empty_runs_and_empty_ranges(cuda_device, small=False):
    """Case 4.  Ranks without rows first, in the middle and last (the `c == 0` skips); shard_bounds with n < 16 W
    (empty owned ranges: check_halo returns early); hand-made zero-length ranges, [N, N) after a rank that ends at N."""
    m, k = 20, 2
    n, world = 1 << 13, 5
    bounds = seams_of(n, world, m + k)
    hay = digits(n, 41)
    for r in (1, 3):
        put(hay, (bounds[r][0] + bounds[r][1]) // 2, TOUCHING)
        put(hay, bounds[r][0] + 8, TOUCHING)
    with local_world(hay, bounds, m + k, cuda_device) as shards:
        got = check_merge(shards, hay, lev(TOUCHING, k), lev_oracle(TOUCHING, hay, k), device=cuda_device)
    assert [len(run) for run in got["runs"]] == [0, 2, 0, 2, 0]
    pat = b"abcdefghijkl"  # m = 12, k = 1: the n-gram route
    for n, world in ((100, 8), (120, 8), (60, 5)):
        bounds = seams_of(n, world, 13)
        assert any(lo == hi for lo, hi in bounds)
        hay = digits(n, n)
        put(hay, 3, pat)
        put(hay, n - 14, pat[:5] + b"X" + pat[6:])
        with local_world(hay, bounds, 13, cuda_device) as shards:
            check_merge(shards, hay, lev(pat, 1), lev_oracle(pat, hay, 1), device=cuda_device)
    n = 160
    hay = digits(n, 43)
    put(hay, 28, TOUCHING)
    put(hay, n - 20, TOUCHING)
    for bounds in ([(0, 0), (0, 48), (48, 48), (48, n), (n, n)], [(0, 48), (48, n), (n, n), (n, n)]):
        with local_world(hay, bounds, m + k, cuda_device) as shards:
            got = check_merge(shards, hay, lev(TOUCHING, k), lev_oracle(TOUCHING, hay, k), device=cuda_device)
            assert got["groups"] == 2 and len(got["runs"][-1]) == 0
            # k >= m (LP route): an empty match (i, i, m) at every i in 0..N, N included, each exactly once
            got = check_merge(shards, hay, lev(b"abc", 3), [(i, i, 3) for i in range(n + 1)], device=cuda_device)
            assert sum(len(run) for run in got["runs"]) == n + 1


@pytest.mark.parametrize("world", [2, 3, 4, 5, 6, 7, 8])
def test_empty_matches_everywhere(cuda_device, world, small=False):
    """Case 4, k >= m in worlds of 2-8: every (i, i, m) once; zero-length hulls are never non-heads."""
    n = 200 if small else 4000
    hay = digits(n, world)
    bounds = seams_of(n, world, 8)
    with local_world(hay, bounds, 8, cuda_device) as shards:
        for pat, k in ((b"abc", 3), (b"a", 5)):
            got = check_merge(shards, hay, lev(pat, k), [(i, i, len(pat)) for i in range(n + 1)], device=cuda_device)
            assert got["groups"] == n + 1 and not got["nonheads"]


@pytest.mark.parametrize("world", [3, 5])
def test_routes_alternate_on_reused_slots(cuda_device, world, small=False):
    """Case 5.  The generic route (n-gram and LP), Hamming, exact and Levenshtein in one world, one after another:
    slots are reused by epoch parity, so every search lands on the slots of the search two before it, written in the
    other mode (consolidated / sorted union) and with more rows than it now brings."""
    from corpus import ASCII, make_corpus
    m, n = 20, (1 << 13 if small else 1 << 16)
    pat, hay, _ = make_corpus(50 + world, n, ASCII, m, 40, 3)
    bounds = seams_of(n, world, m + 4)
    for r in range(1, world):  # copies astride every seam
        put(hay, bounds[r][0] - 7, pat)
        put(hay, bounds[r][0] - 30, pat[:4] + b"#" + pat[5:])
    short = pat[:6]
    steps = [  # (search, oracle, consolidated)
        (lev(pat, 3), lev_oracle(pat, hay, 3), True),
        (lambda h, f: h.search_hamming(pat, 3, f), tup(oracle.substitutions(pat, hay, 3)), False),
        (lambda h, f: h.search_exact(pat, f), [(int(i), int(i) + m, 0) for i in oracle.search_exact(pat, bytes(hay))],
         False),
        (lambda h, f: h.search_generic(pat, 1, 1, 1, 2, f), oracle.find_near_matches(pat, hay, 1, 1, 1, 2), True),
        (lambda h, f: h.search_generic(short, 1, 1, 1, 2, f), oracle.find_near_matches(short, hay, 1, 1, 1, 2), True),
        (lambda h, f: h.search_hamming(pat, 1, f), tup(oracle.substitutions(pat, hay, 1)), False),
        (lev(pat, 1), lev_oracle(pat, hay, 1), True),
    ]
    sizes = []
    with local_world(hay, bounds, m + 4, cuda_device) as shards:
        for search, exp, consolidated in steps:
            got = check_merge(shards, hay, search, exp, consolidated, device=cuda_device)
            sizes.append((consolidated, max(len(run) for run in got["runs"])))
    # a search on the same parity as the one two before it, in the other mode and with fewer rows on some rank
    assert any(sizes[i][0] != sizes[i - 2][0] and sizes[i][1] < sizes[i - 2][1] for i in range(2, len(sizes))), sizes


def capacity_world(n_plants, extra_exact=0, sub=None):
    """World 3: rank 1 owns `n_plants` copies of TOUCHING, 24 bytes apart (the first `n_plants - extra_exact` with the
    byte at `sub` replaced, if `sub` is given), ranks 0 and 2 two copies each; PERIODIC astride both seams for the
    searches after a refusal."""
    lo1 = 1024
    hi1 = (lo1 + 24 * n_plants + 64) // ALIGN * ALIGN
    n = hi1 + 1024
    hay = digits(n, 61)
    for j in range(n_plants):
        plant = bytearray(TOUCHING)
        if sub is not None and j < n_plants - extra_exact:
            plant[sub] = ord("#")
        put(hay, lo1 + 16 + 24 * j, plant)
    for p in (100, 500, hi1 + 100, hi1 + 500):
        put(hay, p, TOUCHING)
    put(hay, lo1 - 7, PERIODIC)
    put(hay, hi1 - 12, PERIODIC)
    return hay, [(0, lo1), (lo1, hi1), (hi1, n)]


def exact(pat):
    return lambda h, f: h.search_exact(pat, f)


def exact_oracle(pat, hay):
    return [(int(i), int(i) + len(pat), 0) for i in oracle.search_exact(pat, bytes(hay))]


def refused_everywhere(shards, search):
    out = search_all(shards, guarded(lambda h: search(h, F.F_GLOBAL).count(F.FINAL)))
    assert all(isinstance(e, F.UnsupportedError) for e in out), out


def test_slot_capacity_edges(cuda_device, small=False):
    """Case 6, rows.  One rank with exactly CAP rows fills its slot (k_push: `nf <= cap`), in both modes: exact copies
    (one row each) and Levenshtein copies (k + 1 = 3 raw records each, 12 288 in all); CAP + 1 rows are refused on
    every rank.  The CAP world also makes the merge's loops wrap: a run of more than 1 024 rows (phase 1 strides) and
    more than W * 1 024 groups (phase 3 strides).  After each refusal the next, smaller searches in the same world are
    right on every rank, in both modes."""
    m, k, world = 20, 2, 3
    hay, bounds = capacity_world(CAP)
    with local_world(hay, bounds, m + k, cuda_device) as shards:
        for search, exp, consolidated in ((exact(TOUCHING), exact_oracle(TOUCHING, hay), False),
                                          (lev(TOUCHING, k), lev_oracle(TOUCHING, hay, k), True)):
            got = check_merge(shards, hay, search, exp, consolidated, device=cuda_device)
            assert [len(run) for run in got["runs"]] == [2, CAP, 2]
            assert got["groups"] > world * THREADS and len(got["runs"][1]) > THREADS
            assert got["raw_counts"][1] == (CAP if not consolidated else CAP * (k + 1))
    hay, bounds = capacity_world(CAP + 1)
    with local_world(hay, bounds, m + k, cuda_device) as shards:
        for search in (exact(TOUCHING), lev(TOUCHING, k), exact(TOUCHING), lev(TOUCHING, k)):
            refused_everywhere(shards, search)
            check_merge(shards, hay, lev(PERIODIC, k), lev_oracle(PERIODIC, hay, k), device=cuda_device)
            check_merge(shards, hay, exact(PERIODIC), exact_oracle(PERIODIC, hay), False, device=cuda_device)


def test_raw_record_edges(cuda_device, small=False):
    """Case 6, raw records.  k = 4 (five 4-grams): a copy with one substitution in its first 4-gram brings 4 raw
    records, an exact copy 5.  CAP such copies on one rank are exactly POST_MAX raw records in CAP groups and merge on
    the device (k_push: `CNT_OUT <= kPostMax`); one exact copy among them makes POST_MAX + 1 and is refused on every
    rank, after which smaller searches in the same world are right."""
    m, k = 20, 4
    hay, bounds = capacity_world(CAP, sub=2)
    with local_world(hay, bounds, m + k, cuda_device) as shards:
        got = check_merge(shards, hay, lev(TOUCHING, k), lev_oracle(TOUCHING, hay, k), device=cuda_device)
        assert got["raw_counts"][1] == POST_MAX and len(got["runs"][1]) == CAP
    hay, bounds = capacity_world(CAP, extra_exact=1, sub=2)
    with local_world(hay, bounds, m + k, cuda_device) as shards:
        assert shards[1].search_levenshtein(TOUCHING, k) is not None and shards[1].debug_counters()[0] == POST_MAX + 1
        refused_everywhere(shards, lev(TOUCHING, k))
        check_merge(shards, hay, lev(PERIODIC, 2), lev_oracle(PERIODIC, hay, 2), device=cuda_device)
        refused_everywhere(shards, lev(TOUCHING, k))
        check_merge(shards, hay, exact(PERIODIC), exact_oracle(PERIODIC, hay), False, device=cuda_device)


def test_world_size_limit(cuda_device, small=False):
    """Case 8.  In-process worlds of more than 16 handles (kMaxWorld) are refused on the host."""
    hs = [F.Haystack.from_host(b"0123456789abcdef", device=cuda_device) for _ in range(17)]
    try:
        with pytest.raises((ValueError, F.UnsupportedError)):
            init_local_world(hs)
    finally:
        for h in hs:
            h.close()
