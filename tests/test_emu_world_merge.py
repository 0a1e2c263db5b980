"""The small cases of test_gpu_world_merge.py replayed on the emulated build (2 SMs), and, without a device, the
restatement those tests compare with: over random geometries (1-8 ranks, arbitrary 16-aligned seams, empty owned
ranges), the restated merge of every rank's own consolidation of the oracle's raw stream (the raw matches whose
anchor the rank owns) equals the oracle's consolidation of the whole sequence.  A mismatch on the device then points
at the device."""
import numpy as np

import oracle
import test_gpu_world_merge as G
from test_emu_kernels import emu_device, emu_lib  # noqa: F401  (fixtures)


def oracle_runs(pat, hay, k, bounds):
    """Every rank's group rows (s, e, d, hull_s, hull_e) from the oracle: the raw matches anchored in its owned range
    (n-gram route: the n-gram hit's index; exact and LP routes: the start), grouped by oracle.consolidate, each group's
    winner its smallest (dist, -length, start) and its hull the members' smallest start and largest end."""
    m, hay = len(pat), bytes(hay)
    if k == 0:
        raw = oracle.levenshtein_raw(pat, hay, 0)
        anchor = raw[:, 0]
    elif m // (k + 1) >= 3:
        raw, _, anchor = oracle.levenshtein_ngrams_raw(pat, hay, k, with_anchor=True)
    else:
        raw = oracle.levenshtein_lp_raw(pat, hay, k)
        anchor = raw[:, 0]
    anchor = np.asarray(anchor)
    runs = []
    for lo, hi in bounds:
        mine = raw[(anchor >= lo) & (anchor < hi)]
        rows = []
        if len(mine):
            winners, groups = oracle.consolidate(mine, with_groups=True)
            for g in np.unique(groups):
                members = mine[groups == g]
                w = min(map(tuple, members.tolist()), key=lambda t: (t[2], -(t[1] - t[0]), t[0]))
                rows.append(w + (int(members[:, 0].min()), int(members[:, 1].max())))
            assert sorted(r[:3] for r in rows) == G.tup(winners)
        rows.sort(key=lambda t: t[3])
        runs.append(np.array(rows, dtype=np.int64).reshape(-1, 5))
    return runs


def random_bounds(rng, n, world):
    """a partition of [0, n) into `world` owned ranges with 16-aligned inner seams, some of them empty"""
    cuts = sorted(int(c) // G.ALIGN * G.ALIGN for c in rng.integers(0, n + 1, size=world - 1))
    if world > 1 and rng.random() < 0.3:
        cuts[int(rng.integers(0, world - 1))] = cuts[0]  # a repeated seam: an empty range in the middle
    edges = [0] + cuts + [n]
    if world > 1 and rng.random() < 0.2:
        edges[-2] = n  # an empty last range [n, n) after a rank that ends at n
    return [(edges[i], edges[i + 1]) for i in range(world)]


def test_restated_merge_equals_the_whole_consolidation():
    rng = np.random.default_rng(901)
    kinds = {"periodic": 0, "nonheads": 0, "equal_hs": 0, "empty": 0}
    for trial in range(200):
        world = int(rng.integers(1, 9))
        m = int(rng.choice([4, 6, 8, 12, 20]))
        k = int(rng.integers(0, min(m - 1, 3) + 1))
        n = int(rng.integers(40, 600))
        alphabet = (b"ACGT", b"abcdefghij", b"ab")[trial % 3]
        hay = np.frombuffer(alphabet, dtype=np.uint8)[rng.integers(0, len(alphabet), size=n)].copy()
        pat = bytes(hay[int(rng.integers(0, n - m)):][:m]) if rng.random() < 0.7 else bytes(G.PERIODIC[:m])
        bounds = random_bounds(rng, n, world)
        runs = oracle_runs(pat, hay, k, bounds)
        got = G.restate(runs)
        assert got["final"] == G.tup(oracle.consolidate(oracle.levenshtein_raw(pat, bytes(hay), k))), \
            (trial, world, m, k, n, bounds)
        kinds["nonheads"] += bool(got["nonheads"])
        kinds["equal_hs"] += bool(G.equal_hull_starts(got["rows"]))
        kinds["empty"] += any(lo == hi for lo, hi in bounds)
    assert kinds["nonheads"] > 30 and kinds["equal_hs"] > 5 and kinds["empty"] > 20, kinds


def test_seam_cases_as_claimed():
    """SEAM_CASES make the per-rank rows the device tests assert (the oracle's side of case 1)"""
    m, k, n = 20, 2, 1024
    for name, (off, run) in G.SEAM_CASES.items():
        hay = G.digits(n, 5)
        G.put(hay, 512 + off, run)
        runs = oracle_runs(G.PERIODIC, hay, k, [(0, 512), (512, n)])
        got = G.restate(runs)
        assert got["final"] == G.lev_oracle(G.PERIODIC, hay, k) and got["groups"] == 1, name
        lower, higher = runs[0][-1], runs[1][0]
        assert (lower[3] == higher[3]) == name.startswith("equal_hs"), (name, lower, higher)


def test_emu_seams(emu_device):
    G.test_equal_hull_starts_and_winner_ties(emu_device, small=True)
    G.test_touching_and_interleaved_hulls(emu_device, small=True)


def test_emu_chains_and_empty_ranges(emu_device):
    G.test_groups_chain_over_every_rank(emu_device, small=True)
    G.test_empty_runs_and_empty_ranges(emu_device, small=True)
    for world in (2, 5, 8):
        G.test_empty_matches_everywhere(emu_device, world, small=True)


def test_emu_routes_alternate(emu_device):
    G.test_routes_alternate_on_reused_slots(emu_device, 3, small=True)


def test_emu_capacity_edges(emu_device):
    G.test_slot_capacity_edges(emu_device, small=True)
    G.test_raw_record_edges(emu_device, small=True)
    G.test_world_size_limit(emu_device, small=True)
