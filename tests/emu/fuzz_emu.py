"""Randomised parity campaign on the CPU emulator: product kernels (tests/emu) vs the CPU oracle.  Developer tool.

    python tests/emu/fuzz_emu.py --seed 1 --trials 400 [--routes world,lev,ham,generic,exact,shard,batch,has]

Far more geometry than the `-m gpu` suite can afford on a GPU budget: tiny and empty sequences, every pattern
length, forced filters, capped work lists (overflow paths), shards with arbitrary seams, grid sizes (FZB_EMU_SMS),
all three Hamming counter layouts.  Every mismatch prints a reproducer line and the run exits non-zero.
"""
import argparse
import os
import sys
import time

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import oracle  # noqa: E402
from conftest import load_emulated_library  # noqa: E402
from corpus import ASCII, DNA, make_corpus  # noqa: E402
from fuzzysearch_b200 import _native as F  # noqa: E402
from parity import tup  # noqa: E402

ALPHABETS = [b"a", b"ab", DNA, b"abcdefgh", ASCII, bytes(range(256))]
if os.environ.get("FZB_FUZZ_ZEROS"):  # the buffers are zero-padded: patterns and text made of zero bytes
    ALPHABETS = [b"\x00", b"\x00\x01", b"\x00\xff\x00\x00", bytes(range(4))]
FAILS = []


def fail(kind, ctx):
    FAILS.append((kind, ctx))
    print("MISMATCH %s %r" % (kind, ctx), flush=True)


def random_case(rng, mmax=255, subs_only=False):
    alphabet = ALPHABETS[int(rng.integers(len(ALPHABETS)))]
    m = int(rng.choice([1, 2, 3, 4, 5, 6, 7, 8, 9, 11, 13, 16, 20, 24, 31, 32, 33, 40, 63, 64, 65, 100, 128, 200, 255]))
    m = min(m, mmax)
    n = int(rng.choice([0, 1, 2, 15, 16, 17, 63, 64, 65, 127, 128, 129, 255, 1000, 4095, 4096, 4097, 16384 + 3,
                        40000, 70001]))
    seed = int(rng.integers(1 << 30))
    if n > 4 * m and rng.integers(4):
        pat, hay, _ = make_corpus(seed, n, alphabet, m, int(rng.integers(1, 12)), int(rng.integers(0, 6)),
                                  subs_only=subs_only, clusters=int(rng.integers(0, 3)))
    else:
        r2 = np.random.default_rng(seed)
        al = np.frombuffer(alphabet, dtype=np.uint8)
        pat = bytes(al[r2.integers(0, len(al), size=m)])
        hay = al[r2.integers(0, len(al), size=n)].copy()
        if n >= m and rng.integers(2):
            pos = int(r2.integers(0, n - m + 1))
            hay[pos:pos + m] = np.frombuffer(pat, dtype=np.uint8)
    return alphabet, pat, hay, seed


def lev_trial(rng):
    alphabet, pat, hay, seed = random_case(rng)
    m = len(pat)
    k = int(rng.integers(0, min(m, 6) + 1)) if rng.integers(4) else int(rng.integers(0, min(m + 2, 41)))
    if k > 0 and m // (k + 1) < 3:  # LP route: exponential candidate lists on repetitive text (reference too)
        k = min(k, 3)
        hay = hay[:3000 if len(alphabet) <= 8 else 30000]
    if len(alphabet) <= 8 and k > 3:
        hay = hay[:3000]
    if len(alphabet) <= 2:
        hay = hay[:1500]
        k = min(k, 2)
    cpu = oracle.levenshtein_raw(pat, hay, k)
    if len(cpu) > 300000:
        return
    want_final = tup(oracle.consolidate(cpu))
    hs = F.Haystack.from_host(hay)
    for flags in (0, F.F_FORCE_DENSE, F.F_FORCE_SAMPLED, F.F_TINY_LIST, F.F_TINY_LIST | F.F_FORCE_DENSE, F.F_FORCE_LP,
                  F.F_FORCE_NGRAMS):
        if flags == F.F_FORCE_LP and (k >= 4 or len(hay) > 5000):
            continue
        if flags == F.F_FORCE_NGRAMS and (k == 0 or m // (k + 1) == 0):
            continue
        ctx = ("lev", seed, len(alphabet), m, k, len(hay), flags, os.environ.get("FZB_EMU_SMS"))
        try:
            res = hs.search_levenshtein(pat, k, flags)
        except F.UnsupportedError:
            continue
        except Exception as e:  # noqa: BLE001
            fail("lev-exception %r" % (e,), ctx)
            continue
        route = res.stats()["route"]
        got = res.triples(F.RAW)
        if flags in (F.F_FORCE_LP, F.F_FORCE_NGRAMS):
            # a forced route emits that route's raw stream; its consolidation is the comparable thing only when
            # the oracle's router picked the same route -- compare against that route's own oracle function
            ref = oracle.levenshtein_lp_raw(pat, hay, k) if route == "lp" else (
                oracle.levenshtein_ngrams_raw(pat, hay, k) if k > 0 else cpu)
            if sorted(got) != sorted(tup(ref)):
                fail("lev-forced-raw", ctx + (route,))
            res.close()
            continue
        if route == "lp" or route == "exact":
            ok = sorted(got) == sorted(tup(cpu))
        else:
            ok = got == tup(cpu)
        if not ok:
            fail("lev-raw", ctx + (route, len(got), len(cpu)))
        elif res.triples(F.FINAL) != want_final:
            fail("lev-final", ctx + (route,))
        res.close()
    hs.close()


def ham_trial(rng):
    alphabet, pat, hay, seed = random_case(rng, subs_only=True)
    m = len(pat)
    k = int(rng.integers(0, 9))
    cpu = tup(oracle.substitutions(pat, hay, k))
    hs = F.Haystack.from_host(hay)
    for layout in ("", "nibble", "sliced3"):
        if layout:
            os.environ["FZB_HAM_COUNTERS"] = layout
        else:
            os.environ.pop("FZB_HAM_COUNTERS", None)
        for flags in (0, F.F_FORCE_DENSE, F.F_TINY_LIST, F.F_FORCE_NGRAMS):
            ctx = ("ham", seed, len(alphabet), m, k, len(hay), flags, layout, os.environ.get("FZB_EMU_SMS"))
            try:
                res = hs.search_hamming(pat, k, flags)
            except F.UnsupportedError:
                continue
            except Exception as e:  # noqa: BLE001
                fail("ham-exception %r" % (e,), ctx)
                continue
            got = res.triples(F.RAW)
            if got != cpu:
                fail("ham", ctx + (res.stats()["route"], len(got), len(cpu)))
            res.close()
    os.environ.pop("FZB_HAM_COUNTERS", None)
    hs.close()


def generic_trial(rng):
    alphabet, pat, hay, seed = random_case(rng, mmax=64)
    m = len(pat)
    subs, ins, dels = (int(x) for x in rng.integers(0, 4, size=3))
    l = int(rng.integers(0, 5)) if rng.integers(3) else None
    try:
        subs, ins, dels, l = oracle.normalize_params(subs, ins, dels, l)
    except Exception:  # noqa: BLE001
        return
    if l == 0:
        return
    hay = hay[:3000 if len(alphabet) <= 4 else 20000]
    if len(alphabet) <= 2:
        hay = hay[:600]
    cpu = oracle.generic_raw(pat, hay, subs, ins, dels, l)
    hs = F.Haystack.from_host(hay)
    for flags in (0, F.F_FORCE_DENSE, F.F_TINY_LIST):
        ctx = ("generic", seed, len(alphabet), m, subs, ins, dels, l, len(hay), flags)
        try:
            res = hs.search_generic(pat, subs, ins, dels, l, flags)
        except F.UnsupportedError:
            continue
        except Exception as e:  # noqa: BLE001
            fail("generic-exception %r" % (e,), ctx)
            continue
        if sorted(res.triples(F.RAW)) != sorted(tup(cpu)):
            fail("generic-raw", ctx + (res.stats()["route"],))
        elif res.triples(F.FINAL) != tup(oracle.consolidate(cpu)):
            fail("generic-final", ctx)
        res.close()
    hs.close()


def exact_trial(rng):
    alphabet, pat, hay, seed = random_case(rng)
    m, n = len(pat), len(hay)
    hs = F.Haystack.from_host(hay)
    for _ in range(4):
        if rng.integers(3) == 0:
            start, end = None, None
        else:
            start = int(rng.integers(0, n + 2))
            end = int(rng.integers(0, n + 2))
        ctx = ("exact", seed, len(alphabet), m, n, start, end)
        want = oracle.search_exact(pat, bytes(hay), 0 if start is None else start, end)
        try:
            res = hs.search_exact(pat, 0, start, end) if start is not None else hs.search_exact(pat)
        except Exception as e:  # noqa: BLE001
            fail("exact-exception %r" % (e,), ctx)
            continue
        got = [s for s, _, _ in res.triples(F.RAW)]
        if got != [int(x) for x in want]:
            fail("exact", ctx + (len(got), len(want)))
        res.close()
    hs.close()


def shard_trial(rng):
    alphabet, pat, hay, seed = random_case(rng, mmax=64)
    m, n = len(pat), len(hay)
    if n < 64:
        return
    k = int(rng.integers(0, min(m, 4) + 1))
    if k > 0 and m // (k + 1) < 3:
        k = min(k, 2)
        hay = hay[:4000]
        n = len(hay)
    if len(alphabet) <= 2:
        hay = hay[:1500]
        n = len(hay)
        k = min(k, 2)
    nshards = int(rng.integers(2, 6))
    cuts = sorted(set(int(x) // 16 * 16 for x in rng.integers(1, n, size=nshards - 1)))
    bounds = [0] + [c for c in cuts if 0 < c < n] + [n]
    halo = m + k
    whole = sorted(tup(oracle.levenshtein_raw(pat, hay, k)))
    if len(whole) > 200000:
        return
    ham_whole = tup(oracle.substitutions(pat, hay, k))
    got, ham = [], []
    for i in range(len(bounds) - 1):
        lo, hi = bounds[i], bounds[i + 1]
        blo = max(0, lo - halo - int(rng.integers(0, 40))) // 16 * 16
        bhi = min(n, hi + halo + int(rng.integers(0, 40)))
        hs = F.Haystack.from_host(hay[blo:bhi], buf_lo=blo, global_len=n, own_lo=lo, own_hi=hi)
        res = hs.search_levenshtein(pat, k, F.F_NO_FINAL)
        got += res.triples(F.RAW)
        res.close()
        res = hs.search_hamming(pat, k)
        ham += res.triples(F.RAW)
        res.close()
        hs.close()
    ctx = ("shard", seed, len(alphabet), m, k, n, bounds)
    if sorted(got) != whole:
        fail("shard-lev", ctx + (len(got), len(whole)))
    if sorted(ham) != ham_whole:
        fail("shard-ham", ctx + (len(ham), len(ham_whole)))


def batch_trial(rng):
    alphabet = ALPHABETS[int(rng.integers(2, len(ALPHABETS)))]
    n = int(rng.choice([0, 100, 5000, 60000]))
    if len(alphabet) <= 4:
        n = min(n, 5000)
    seed = int(rng.integers(1 << 30))
    r2 = np.random.default_rng(seed)
    al = np.frombuffer(alphabet, dtype=np.uint8)
    hay = al[r2.integers(0, len(al), size=n)].copy()
    pats, ks = [], []
    for _ in range(int(rng.integers(1, 40))):
        m = int(rng.integers(1, 80))
        k = int(rng.integers(0, 5))
        if k > 0 and m // (k + 1) < 3 and len(alphabet) <= 8:
            k = min(k, 2)
        p = bytes(al[r2.integers(0, len(al), size=m)])
        if n > 2 * m and rng.integers(3):  # plant it, with some edits
            pos = int(r2.integers(0, n - m))
            v = bytearray(p)
            for _e in range(int(rng.integers(0, k + 2))):
                if v:
                    v[int(r2.integers(len(v)))] = int(al[int(r2.integers(len(al)))])
            hay[pos:pos + len(v)] = np.frombuffer(bytes(v), dtype=np.uint8)
        pats.append(p)
        ks.append(k)
    if rng.integers(3) == 0 and pats:
        pats.append(pats[0])  # duplicate pattern
        ks.append(ks[0])
    hs = F.Haystack.from_host(hay)
    ctx = ("batch", seed, len(alphabet), n, len(pats))
    try:
        results, _ = hs.search_levenshtein_batch(pats, ks)
    except F.UnsupportedError:
        hs.close()
        return
    except Exception as e:  # noqa: BLE001
        fail("batch-exception %r" % (e,), ctx)
        hs.close()
        return
    for i, (p, k, res) in enumerate(zip(pats, ks, results)):
        cpu = oracle.levenshtein_raw(p, hay, k)
        want = tup(oracle.consolidate(cpu))
        got = res.triples(F.FINAL)
        if got != want:
            fail("batch", ctx + (i, len(p), k, len(got), len(want)))
        # k == 0: find_near_matches_batch() hands out the RAW stream (ExactSearch does not consolidate)
        if k == 0 and sorted(res.triples(F.RAW)) != sorted(tup(cpu)):
            fail("batch-raw-k0", ctx + (i, len(p)))
        res.close()
    hs.close()


def has_trial(rng):
    alphabet, pat, hay, seed = random_case(rng, mmax=64)
    m = len(pat)
    big = 1 << 30
    mode = int(rng.integers(3))
    if mode == 0:
        k = int(rng.integers(0, min(m, 4) + 1))
        if k > 0 and m // (k + 1) < 3:
            hay = hay[:3000]
        lim = (big, big, big, k)
        want = len(oracle.levenshtein_raw(pat, hay, k)) > 0
    elif mode == 1:
        k = int(rng.integers(0, 6))
        lim = (k, 0, 0, k)
        want = len(oracle.substitutions(pat, hay, k)) > 0
    else:
        subs, ins, dels = (int(x) for x in rng.integers(0, 3, size=3))
        l = int(rng.integers(1, 4))
        subs, ins, dels, l = oracle.normalize_params(subs, ins, dels, l)
        if l == 0:
            return
        hay = hay[:5000]
        lim = (subs, ins, dels, l)
        want = len(oracle.find_near_matches(pat, hay, subs, ins, dels, l)) > 0
    hs = F.Haystack.from_host(hay)
    chunk = int(rng.choice([0, 128, 512, 4096]))  # chunked early termination: seams at small sizes
    if chunk:
        os.environ["FZB_HAS_CHUNK_BYTES"] = str(chunk)
    else:
        os.environ.pop("FZB_HAS_CHUNK_BYTES", None)
    try:
        got = hs.has_near_match(pat, *lim)
        if bool(got) != want:
            fail("has", ("has", seed, len(alphabet), m, len(hay), lim, got, want, chunk))
    except F.UnsupportedError:
        pass
    except Exception as e:  # noqa: BLE001
        fail("has-exception %r" % (e,), ("has", seed, m, len(hay), lim))
    os.environ.pop("FZB_HAS_CHUNK_BYTES", None)
    hs.close()


def world_trial(rng):
    """In-process world (one host thread per shard): the k_push / k_merge reduction vs the oracle's global list."""
    from fuzzysearch_b200.sharding import init_local_world, search_all, shard_bounds
    alphabet = ALPHABETS[int(rng.integers(2, len(ALPHABETS)))]
    world = int(rng.integers(1, 9))
    m = int(rng.choice([3, 5, 8, 12, 20, 33, 64]))
    k = int(rng.integers(0, min(m - 1, 4) + 1))
    n = int(rng.choice([64, 300, 4096, 4097, 70000]))
    if k > 0 and m // (k + 1) < 3:
        k = min(k, 2)
        n = min(n, 4096)
    if len(alphabet) <= 4:
        n = min(n, 4096)
    n = max(n, world * 32)
    seed = int(rng.integers(1 << 30))
    pat, hay, _ = make_corpus(seed, n, alphabet, m, int(rng.integers(1, 12)), k + 1, clusters=int(rng.integers(0, 4)))
    halo = m + max(k, 3)
    for r in range(1, world):  # something straddling every seam
        seam = shard_bounds(n, world, r, halo)[2]
        pos = seam - int(rng.integers(0, m + 1))
        if 0 <= pos and pos + m <= n:
            hay[pos:pos + m] = np.frombuffer(pat, dtype=np.uint8)
    shards = []
    for r in range(world):
        blo, bhi, lo, hi = shard_bounds(n, world, r, halo)
        shards.append(F.Haystack.from_host(hay[blo:bhi], buf_lo=blo, global_len=n, own_lo=lo, own_hi=hi))
    ctx = ("world", seed, len(alphabet), world, m, k, n)
    try:
        init_local_world(shards)
        want = {"lev": tup(oracle.consolidate(oracle.levenshtein_raw(pat, hay, k))),  # C-ABI level: FINAL of k == 0 too
                "ham": tup(oracle.substitutions(pat, hay, min(k, 3))),
                "exact": [(int(i), int(i) + m, 0) for i in oracle.search_exact(pat, bytes(hay))]}
        calls = {"lev": lambda h: h.search_levenshtein(pat, k, F.F_GLOBAL).triples(F.FINAL),
                 "ham": lambda h: h.search_hamming(pat, min(k, 3), F.F_GLOBAL).triples(F.FINAL),
                 "exact": lambda h: h.search_exact(pat, F.F_GLOBAL).triples(F.FINAL)}
        for name in ("lev", "ham", "exact", "lev"):
            try:
                got = search_all(shards, calls[name])
            except F.UnsupportedError:
                continue  # more groups than a peer slot holds: the in-process world has no staged path
            for r in range(world):
                if got[r] != want[name]:
                    fail("world-" + name, ctx + (r, len(got[r]), len(want[name])))
                    break
    except Exception as e:  # noqa: BLE001
        fail("world-exception %r" % (e,), ctx)
    finally:
        for h in shards:
            h.close()


TRIALS = {"world": world_trial, "lev": lev_trial, "ham": ham_trial, "generic": generic_trial, "exact": exact_trial, "shard": shard_trial,
          "batch": batch_trial, "has": has_trial}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seed", type=int, default=1)
    ap.add_argument("--trials", type=int, default=200)
    ap.add_argument("--routes", default=",".join(TRIALS))
    ap.add_argument("--seconds", type=float, default=0, help="stop after this many seconds (0 = run all trials)")
    a = ap.parse_args()
    F._lib = load_emulated_library()
    rng = np.random.default_rng(a.seed)
    routes = a.routes.split(",")
    t0 = time.time()
    done = 0
    for t in range(a.trials):
        os.environ["FZB_EMU_SMS"] = str(int(rng.choice([1, 2, 4, 7])))
        for r in routes:
            TRIALS[r](rng)
        done += 1
        if a.seconds and time.time() - t0 > a.seconds:
            break
        if t % 20 == 19:
            print("trial %d  %.0fs  mismatches %d" % (t + 1, time.time() - t0, len(FAILS)), flush=True)
    print("done: %d trials x %s in %.0fs, %d mismatches" % (done, routes, time.time() - t0, len(FAILS)))
    return 1 if FAILS else 0


if __name__ == "__main__":
    sys.exit(main())
