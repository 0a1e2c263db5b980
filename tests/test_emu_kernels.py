"""The product's CUDA sources replayed on the CPU: `pytest -m "not gpu"` coverage of the KERNELS and of api.cu.

tests/emu compiles fuzzysearch_b200/csrc (api.cu and every *.cuh, the code that ships) against a small CUDA
execution-model emulator -- fibers for threads, rendezvous for the warp collectives, TMA / mbarrier restated -- into
tests/emu/_build/libfuzzb200_emu.so with the same C-ABI.  The tests below bind it in place of libfuzzb200.so and run
the bodies of the `-m gpu` parity tests (same functions, same oracle, same fixtures) at the sizes a CPU can do in
seconds.  It proves kernel LOGIC and host logic -- filters lose no match, work lists and overflow paths, bit-parallel
expansions, consolidation, batches, wide symbols, file loops, locking, the peer-memory reduction of in-process
multi-shard worlds -- not timing, memory-model behaviour, CUDA IPC or NCCL (those need a real GPU:
tests/test_gpu_global.py, bench.py).  The emulated library is test
infrastructure: nothing in the product can load it.

`FZB_TEST_BACKEND=emu python -m pytest tests -m gpu` replays the whole GPU suite this way (minutes), and
`python tests/emu/fuzz_emu.py` runs a randomised campaign far beyond what fits a GPU budget.
"""
import ctypes
import gc
import inspect

import pytest

import conftest
import test_gpu_batch
import test_gpu_batch_edges
import test_gpu_expand
import test_gpu_file
import test_gpu_fuzz
import test_gpu_global
import test_gpu_golden
import test_gpu_lp_generic_edges
import test_gpu_ngram_edges
import test_gpu_oracle
import test_gpu_python_api
import test_gpu_symbols
from fuzzysearch_b200 import _native, search


@pytest.fixture(scope="module")
def emu_lib():
    return conftest.load_emulated_library()


@pytest.fixture()
def emu_device(emu_lib, monkeypatch):
    monkeypatch.setattr(_native, "_lib", emu_lib)
    monkeypatch.setenv("FZB_EMU_SMS", "2")  # small grids: the replays are dominated by per-launch fiber set-up
    saved = dict(search._WORKSPACE)
    search._WORKSPACE.clear()
    yield 0
    search.release_workspace()
    gc.collect()  # every handle of the emulated library dies while it is still the bound one
    search._WORKSPACE.update(saved)


def _cases(func):
    """Expand the @pytest.mark.parametrize marks of a gpu test function into keyword dicts."""
    out = [{}]
    for mark in getattr(func, "pytestmark", []):
        if mark.name != "parametrize":
            continue
        names = [a.strip() for a in mark.args[0].split(",")]
        new = []
        for base in out:
            for values in mark.args[1]:
                if len(names) == 1:
                    values = (values,)
                d = dict(base)
                d.update(zip(names, values))
                new.append(d)
        out = new
    return out


def _run(func, device, **extra):
    for kw in _cases(func):
        kw.update(extra)
        func(device, **kw)


def test_emulator_is_the_product_source(emu_lib):
    """Same exported C-ABI as the header declares, and it says it is an emulator only through the device name."""
    for name in _native.SYMBOLS:
        assert hasattr(emu_lib, name), name
    assert emu_lib.fzb_device_count() == 1


def test_emu_ngram_route_vs_oracle(emu_device):
    _run(test_gpu_oracle.test_levenshtein_ngrams_matches_oracle, emu_device)


def test_emu_hamming_lp_generic_vs_oracle(emu_device):
    _run(test_gpu_oracle.test_hamming_matches_oracle, emu_device)
    _run(test_gpu_oracle.test_levenshtein_lp_matches_oracle, emu_device)
    _run(test_gpu_oracle.test_generic_matches_oracle, emu_device)


def test_emu_shards_edge_cases_python_surface(emu_device):
    _run(test_gpu_oracle.test_sharded_union_equals_whole, emu_device)
    test_gpu_oracle.test_edge_cases(emu_device)
    test_gpu_oracle.test_python_surface_variants(emu_device)
    test_gpu_oracle.test_positions_are_64_bit_everywhere(emu_device)


def test_emu_random_sweeps(emu_device):
    test_gpu_fuzz.test_levenshtein_random_sweep(emu_device)
    test_gpu_fuzz.test_hamming_random_sweep(emu_device)
    test_gpu_fuzz.test_generic_random_sweep(emu_device)


def test_emu_expansion_kernels(emu_device):
    test_gpu_expand.test_expand_golden_records(emu_device)
    test_gpu_expand.test_expand_quirk_vectors(emu_device)
    test_gpu_expand.test_expand_fuzz_vs_oracle(emu_device)


def test_emu_reference_suite_calls(emu_device):
    test_gpu_golden.test_gpu_replays_reference_suite_calls(emu_device)
    test_gpu_golden.test_gpu_module_level_route_functions(emu_device)


def test_emu_batches(emu_device):
    test_gpu_batch.test_batch_matches_oracle(emu_device)
    test_gpu_batch.test_batch_shared_scan_edge_cases(emu_device)
    test_gpu_batch.test_batch_lp_pass_with_large_budgets(emu_device)
    test_gpu_batch.test_batch_dense_pass_flushes_and_overflows_its_cta_buffer(emu_device)


def test_emu_batch_edges(emu_device):
    """Batches on shards at 64-bit offsets, sharded unions, past the pass limits, through the overflow fallbacks
    and across the LP chunk seams (the 600 MiB seam test needs a real GPU)."""
    test_gpu_batch_edges.test_batch_at_64_bit_offsets(emu_device)
    _run(test_gpu_batch_edges.test_batch_sharded_union_equals_whole, emu_device)
    _run(test_gpu_batch_edges.test_batch_lp_pass_limits, emu_device)
    test_gpu_batch_edges.test_batch_two_q_sample_passes(emu_device)
    test_gpu_batch_edges.test_batch_gram_with_more_than_255_postings(emu_device)
    test_gpu_batch_edges.test_batch_overflow_fallbacks(emu_device)
    test_gpu_batch_edges.test_batch_lp_chunk_seams(emu_device)


def test_emu_lp_generic_edges(emu_device):
    """The LP and generic routes at their limits: every k_lp_verify mode, streaming windows 47-50, the survivor-list
    overflow (FZB_F_TINY_LIST), candidate-list growth and the 16 384 limit, 6-bit counters at 63, clipped n-gram
    windows, sharded unions and offsets up to 2^44."""
    _run(test_gpu_lp_generic_edges.test_lp_verify_and_window_boundaries, emu_device)
    _run(test_gpu_lp_generic_edges.test_lp_scan_look_ahead, emu_device)
    test_gpu_lp_generic_edges.test_lp_survivor_list_overflow(emu_device)
    _run(test_gpu_lp_generic_edges.test_candidate_list_growth, emu_device)
    test_gpu_lp_generic_edges.test_candidate_limit(emu_device)
    _run(test_gpu_lp_generic_edges.test_generic_counters_at_63, emu_device)
    test_gpu_lp_generic_edges.test_generic_lowering_rule(emu_device)
    _run(test_gpu_lp_generic_edges.test_generic_ngram_windows_at_global_ends, emu_device)
    _run(test_gpu_lp_generic_edges.test_lp_generic_sharded_union_equals_whole, emu_device)
    test_gpu_lp_generic_edges.test_lp_generic_at_64_bit_offsets(emu_device)


def test_emu_ngram_edges(emu_device):
    """The n-gram Levenshtein route at its margins: the q-sample lemma, every byte offset of the dense filters, the
    verify modes and the hit slot, the hand-over to the host and to a larger output buffer, sharded unions."""
    _run(test_gpu_ngram_edges.test_sampled_filter_at_the_lemma_margin, emu_device)
    _run(test_gpu_ngram_edges.test_dense_filters_at_every_byte_offset, emu_device)
    _run(test_gpu_ngram_edges.test_verify_kernels_at_their_limits, emu_device)
    test_gpu_ngram_edges.test_same_match_through_several_ngrams(emu_device)
    _run(test_gpu_ngram_edges.test_post_hand_over, emu_device)
    _run(test_gpu_ngram_edges.test_post_groups_across_rounds, emu_device)
    _run(test_gpu_ngram_edges.test_output_buffer_growth, emu_device)
    _run(test_gpu_ngram_edges.test_ngram_sharded_union_equals_whole, emu_device)


def test_emu_file_search(emu_device, tmp_path):
    for i, kw in enumerate(_cases(test_gpu_file.test_match_split_between_chunks)):
        if kw["chunk_size"] < 1000:
            continue  # hundreds of tiny searches: left to the full replay
        d = tmp_path / ("c%d" % i)
        d.mkdir()
        test_gpu_file.test_match_split_between_chunks(emu_device, tmp_path=d, **kw)
    test_gpu_file.test_file_random_corpus(emu_device, tmp_path)


def test_emu_has_near_match_chunk_seams(emu_device, monkeypatch):
    test_gpu_python_api.test_has_near_match_chunk_seams_at_small_scale(emu_device, monkeypatch)


def test_emu_threads_and_has_near_match(emu_device):
    test_gpu_python_api.test_find_near_matches_is_thread_safe(emu_device)
    test_gpu_python_api.test_threads_share_one_resident_sequence(emu_device)
    test_gpu_python_api.test_has_near_match_all_routes_vs_oracle(emu_device)


def test_emu_multi_shard_worlds(emu_device):
    """The multi-GPU reduction (k_push -> k_merge over the peers' receive areas, grid-wide barrier included) in
    in-process worlds of 2, 3, 4 and 8 shards, one host thread per shard: every rank must hold the oracle's
    global list.  (CUDA IPC / NCCL bootstrap and the staged path need real devices: tests/test_gpu_global.py.)"""
    for kw in _cases(test_gpu_global.test_multi_rank_world_on_one_gpu):
        if kw["world"] < 8:  # (the 8-shard, 2 MiB case: FZB_TEST_BACKEND=emu python -m pytest tests/test_gpu_global.py)
            test_gpu_global.test_multi_rank_world_on_one_gpu(emu_device, **kw)
    test_gpu_global.test_multi_rank_lp_and_dna_routes(emu_device)
    _run(test_gpu_global.test_seam_rows_interleave_between_runs, emu_device)
    test_gpu_global.test_local_world_refuses_what_needs_the_staged_path(emu_device)


def test_emu_wide_symbols(emu_device, tmp_path):
    for kw in _cases(test_gpu_symbols.test_device_reduction_of_code_units):
        if kw["n"] <= 1 << 16:
            test_gpu_symbols.test_device_reduction_of_code_units(emu_device, **kw)
    test_gpu_symbols.test_resident_wide_sequence_and_batches(emu_device)
    test_gpu_symbols.test_items_resident_and_mixed_types(emu_device)
    sig = inspect.signature(test_gpu_symbols.test_wide_cases_of_the_reference_suite)
    assert list(sig.parameters) == ["cuda_device", "tmp_path"]
    test_gpu_symbols.test_wide_cases_of_the_reference_suite(emu_device, tmp_path)


def test_emu_allocation_failures_surface_cleanly(emu_device, monkeypatch):
    """Fault injection (FZB_EMU_FAIL_ALLOC=N: the N-th device / pinned allocation fails once): every failure must
    come back as CudaError through the C-ABI -- no crash, no wrong answer -- and the library must be sane afterwards
    (an out-of-memory search on a shared box is not allowed to poison the process), with nothing leaked."""
    import os

    import numpy as np  # noqa: F401

    import oracle
    from corpus import ASCII, DNA, make_corpus
    from parity import tup
    F = _native
    pat, hay, _ = make_corpus(5, 1 << 13, ASCII, 20, 8, 3)
    patd, hayd, _ = make_corpus(6, 1 << 11, DNA, 20, 8, 3)

    def searches():
        hs = F.Haystack.from_host(hay)
        out = [hs.search_levenshtein(pat, 2).triples(F.FINAL), hs.search_hamming(pat, 3).triples(F.FINAL),
               hs.search_levenshtein(pat[:8], 3).triples(F.FINAL), hs.search_generic(pat, 1, 2, 1, 2).triples(F.FINAL)]
        hs2 = F.Haystack.from_host(hayd)
        out.append(hs2.search_levenshtein(patd, 2).triples(F.FINAL))
        out.append(hs.has_near_match(pat, 1 << 29, 1 << 29, 1 << 29, 2))
        hs2.close()
        hs.close()
        return out

    def batch():
        hs = F.Haystack.from_host(hay)
        res, _ = hs.search_levenshtein_batch([pat, pat[:30], pat[2:12], pat[:9], pat[1:9]], [2, 1, 1, 3, 3])
        out = [r.triples(F.FINAL) for r in res]
        hs.close()
        return out

    assert searches()[0] == tup(oracle.consolidate(oracle.levenshtein_raw(pat, hay, 2)))
    live = _native.lib().fzb_emu_live_allocations  # emulator-only export: device + pinned allocations not yet freed
    live.restype = ctypes.c_long
    for scenario, upto, at_least in ((searches, 60, 15), (batch, 40, 10)):
        good = scenario()
        gc.collect()
        baseline = live()
        raised = 0
        for nth in range(1, upto):
            monkeypatch.setenv("FZB_EMU_FAIL_ALLOC", str(nth))
            failed = False
            try:
                assert scenario() == good, nth   # no such allocation, or an optional buffer
            except F.CudaError:
                failed = True  # (the traceback keeps the scenario's handles alive until the handler is left)
            monkeypatch.setenv("FZB_EMU_FAIL_ALLOC", "")
            if failed:
                raised += 1
                gc.collect()  # the handles of the failed scenario are gone: whatever it allocated must be, too
                assert live() == baseline, ("leak on the error path of allocation", nth)
                assert scenario() == good, ("library state after a failed allocation", nth)
        assert raised >= at_least, (scenario.__name__, raised)
    assert "FZB_EMU_FAIL_ALLOC" in os.environ


def _alloc_failure_scenarios():
    """name -> (open() -> state, call(state) -> comparable answer).  Each call reaches allocations a handle makes
    after it was created: lazily allocated buffer groups and grow paths."""
    import numpy as np

    from corpus import ASCII, DNA, make_corpus
    from fuzzysearch_b200.sharding import init_local_world, search_all, shard_bounds
    F = _native
    rng = np.random.default_rng(7)
    dna = bytes(rng.choice(np.frombuffer(DNA, np.uint8), size=1 << 17))
    _, text, _ = make_corpus(8, 1 << 13, ASCII, 20, 8, 3)
    text = text.tobytes()
    lp_pat, lp_hay, _ = make_corpus(2, 300, DNA, 16, 4, 8)  # > 256 live candidates at some start (test_gpu_lp_generic_edges)

    def routes(results):
        return [(r.stats()["route"], r.triples(F.FINAL)) for r in results[0]]

    def lev_batch(hs):  # two q-sample patterns, two for the dense pass, two for the LP pass
        pats = [text[100:130], text[300:330], text[500:511], text[700:710], text[900:908], text[1100:1109]]
        return routes(hs.search_levenshtein_batch(pats, [1, 2, 1, 1, 3, 3]))

    def ham_batch(hay, m, k):
        return lambda hs: routes(hs.search_hamming_batch([hay[p:p + m] for p in range(64, 64 + 6 * 97, 97)], [k] * 6))

    def world_open():
        shards = []
        for r in range(2):
            blo, bhi, lo, hi = shard_bounds(len(text), 2, r, 64)
            shards.append(F.Haystack.from_host(text[blo:bhi], buf_lo=blo, global_len=len(text), own_lo=lo, own_hi=hi))
        return shards

    def world_call(shards):
        init_local_world(shards)
        return search_all(shards, lambda h: h.search_levenshtein(text[2000:2020], 2, F.F_GLOBAL).triples(F.FINAL))

    def symbols(hs):
        hs.upload_symbols(np.arange(3000, dtype=np.uint32) % 97 + 70000, [70001, 70005, 70020])
        return hs.read(0, len(hs))

    def synthetic(hs):
        hs.fill_synthetic(b"ACGT", 11)
        return hs.read(0, len(hs))

    one = lambda hay: lambda: F.Haystack.from_host(hay)  # noqa: E731
    return {
        "output growth": (one(dna), lambda hs: (hs.search_levenshtein(b"ACGTAC", 3).count(F.RAW),
                                                 hs.search_levenshtein(b"ACGTAC", 3).triples(F.FINAL))),
        "lp scratch growth": (one(lp_hay), lambda hs: hs.search_levenshtein(lp_pat, 7, F.F_FORCE_LP).triples(F.FINAL)),
        "levenshtein batch": (one(text), lev_batch),
        "hamming batch text": (one(text), ham_batch(text, 20, 2)),
        "hamming batch dna": (one(dna[:1 << 14]), ham_batch(dna, 32, 3)),
        "has_near_match": (one(text), lambda hs: [hs.has_near_match(text[40:60], 0, 0, 2, 2),
                                                  hs.has_near_match(b"qqqqqqqqqqqqqq", 1, 1, 1, 2)]),
        "local world": (world_open, world_call),
        "upload_symbols": (lambda: F.Haystack.alloc(4096), symbols),
        "fill_synthetic": (lambda: F.Haystack.alloc(1000), synthetic),
    }


def _replay_allocation_failures(name, upto):
    """Child-process side of test_emu_allocation_failures_leave_the_handle_usable: for nth = 1 .. upto - 1, make the
    scenario's call on a handle that outlives the failure with the nth allocation failing, repeat it on that handle
    without the failure, close it and count what is still allocated.  Prints one line per nth."""
    import os

    F = _native
    F._lib = conftest.load_emulated_library()
    live = F._lib.fzb_emu_live_allocations
    live.restype = ctypes.c_long
    open_, call = _alloc_failure_scenarios()[name]

    def close(state):
        for h in state if isinstance(state, list) else [state]:
            h.close()

    state = open_()
    good = call(state)
    close(state)
    gc.collect()
    baseline = live()
    for nth in range(1, upto):
        state = open_()
        os.environ["FZB_EMU_FAIL_ALLOC"] = str(nth)
        try:
            failed, got = False, call(state)
        except F.CudaError:
            failed, got = True, None
        finally:
            os.environ["FZB_EMU_FAIL_ALLOC"] = ""
        assert failed or got == good, (name, nth, "wrong answer")
        assert call(state) == good, (name, nth, "wrong answer on the handle that saw the failure")
        close(state)
        gc.collect()
        assert live() == baseline, (name, nth, "leak")
        print("%s nth=%d %s" % (name, nth, "raised" if failed else "ok"), flush=True)


@pytest.mark.parametrize("name,upto,failing", [
    ("output growth", 5, 3),        # LP list, candidate lists, the output buffer grown past 65 536 records
    ("lp scratch growth", 5, 3),    # LP list, candidate lists at 256, grown to 2 048 entries
    ("levenshtein batch", 15, 13),  # batch tables (7), dense hit list, LP batch buffers (4), candidate lists
    ("hamming batch text", 9, 7),   # batch tables
    ("hamming batch dna", 9, 7),
    ("has_near_match", 3, 1),
    ("local world", 14, 12),        # the peer-memory buffers of both handles
    ("upload_symbols", 4, 2),       # alphabet, chunk buffer
    ("fill_synthetic", 3, 1),       # alphabet
])
def test_emu_allocation_failures_leave_the_handle_usable(emu_lib, name, upto, failing):
    """A failed allocation in a call on a live handle (FZB_EMU_FAIL_ALLOC=N, for every N the call reaches) comes back
    as CudaError, and the same call on the same handle then returns the right answer: no buffer group is left half
    built and no grown buffer is lost.  Each scenario replays in a child process, so a handle left pointing at
    missing memory fails this test by name instead of killing the session.  `failing`: allocations the call makes;
    the last N makes none fail."""
    import os
    import subprocess
    import sys
    code = "import sys; sys.path[:0] = %r; import test_emu_kernels as t; t._replay_allocation_failures(%r, %d)" % (
        [conftest.ROOT, os.path.join(conftest.ROOT, "tests")], name, upto)
    env = dict(os.environ, FZB_EMU_SMS="2", FZB_EMU_FAIL_ALLOC="")
    p = subprocess.run([sys.executable] + (["-s"] if sys.flags.no_user_site else []) + ["-c", code], env=env,
                       capture_output=True, text=True, timeout=1800)
    lines = p.stdout.split("\n")
    assert p.returncode == 0, (name, "exit %d" % p.returncode, lines[-6:], p.stderr[-3000:])
    raised = [ln for ln in lines if ln.endswith(" raised")]
    assert len(raised) == failing, (name, lines)
    assert lines[-2].endswith("nth=%d ok" % (upto - 1)), (name, lines)  # the scenario's last allocation was reached


def test_emulator_racecheck_sees_a_missing_barrier():
    """tests/emu/selftest: under the emulator's ThreadSanitizer mode a kernel without its __syncthreads() and one
    whose threads all store to one global word are reported; the correct twins (__syncthreads, __syncwarp within a
    warp) are not.  (The product kernels run clean in that mode: tests/emu/README.md.)"""
    import importlib.util
    import os
    import subprocess
    if not os.path.exists(subprocess.run(["/usr/bin/gcc", "-print-file-name=libtsan.so"], capture_output=True,
                                         text=True).stdout.strip() or "/nonexistent"):
        pytest.skip("libtsan not installed")
    spec = importlib.util.spec_from_file_location("fzb_emu_selftest", os.path.join(conftest.ROOT, "tests", "emu",
                                                                                    "selftest.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    reports = mod.run()
    assert reports[(0, False)] == 0 and reports[(2, False)] == 0 and reports[(0, True)] == 0, reports
    assert reports[(1, False)] > 0 and reports[(3, False)] > 0, reports
    # two CTAs storing to one word: invisible while CTAs are ordered, reported in grid mode (unordered CTAs)
    assert reports[(4, False)] == 0 and reports[(4, True)] > 0, reports
