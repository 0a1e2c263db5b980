"""The five scans that batches share, at the geometry of their tiles, buffers and chunks: k_filter_multi (q-sample
pass), k_filter_mdense (n-gram prefix pass), k_filter_mdense2 (2-bit n-gram pass on DNA), k_ham_batch_scan
(substitutions-only pass, text and 2-bit keys) and k_lp_scan_multi (LP pass).

What a scan hands to verification is counted in stats()["n_candidates"], which a pass puts on its first pattern.  The
tests restate that count in numpy from the definition of each filter -- not from its code -- and compare it exactly:
  q-sample  distinct (pattern, granule) pairs: every 4-byte word at 4w < round_up(buf_len, 16) (the zero padding of
            the last vector included) that equals P[o:o+4] marks the granules of the anchors [g-o-K, g-o+K+m-L],
            clipped to the own range; K = k (Levenshtein) or 2k (generic).
  prefix,   hits (pattern, n-gram j, g): g in the own range (and the chunk), g + L <= N and H[g:g+L] == P[jL:(j+1)L];
  2-bit     one per posting, so repeated n-grams and duplicate patterns count each time.
  Hamming   (pattern, piece j, g) with g < buf_len whose key equals piece j's and st = g - jL in the own range with
            st + m <= N: text keys are the first min(L, 4) bytes (zero padding past the end), 2-bit keys the codes of
            min(L, 8) symbols under the pass's code table (two_bit_code).  Counted before verification.
  LP        survivors (pattern, s): s in the own range and below lim = min(N, buf_lo + buf_len), H[s] in
            P[:min(k, m-1)+1] (any byte for generic patterns), and at least m - k bytes of H[s : min(s+wmax, lim))
            occur in P; wmax is the longest m + k of the pass.  Summed over chunks.
Every case also checks that each pattern rode the intended pass and that pass alone (one scan, on the first pattern),
and that each pattern's RAW and FINAL lists equal its single search on the same handle and the oracle where the size
allows.  `small` replays every body on the emulated device (2 SMs) in tests/test_emu_batch_scans.py."""
import numpy as np
import pytest

import oracle
from corpus import ASCII, DNA, mutate
from fuzzysearch_b200 import _native as F
from parity import tup

pytestmark = pytest.mark.gpu

SAMPLED, DENSE, LP, HAM = "ngrams/sampled-filter", "ngrams/dense-filter", "lp", "hamming/batch-scan"
GSAMPLED, GLP = "generic-ngrams/batch-scan", "generic-lp/batch-scan"
TILE = 4096 * 16          # k_filter_multi / _mdense / _mdense2 / k_ham_batch_scan: 1024 threads x 4 vectors
WARP = 32 * 16            # the 16-byte vectors of one warp: lane 31 loads its neighbour words from the next vector
LP_TILE = 256 * 128       # k_lp_scan_multi: 256 threads x a run of 128 starts
SMS, EMU_SMS = 132, 2     # an H100's SMs; the emulated device's (FZB_EMU_SMS)
TINY_CHUNK = 3000         # FZB_F_TINY_LIST: positions per chunk of the 2-bit and LP passes
HASH = 0x9E3779B1         # kernels.cuh: kHashMul (level 1 of the q-sample and text-key tables)
HASH_INV = pow(HASH, -1, 1 << 32)
ORACLE_MAX = 1 << 18      # longer buffers are checked against the single search only


# ------------------------------------------------------------------------------------------------ restatements
def u8(x):
    return np.frombuffer(bytes(x), dtype=np.uint8) if not isinstance(x, np.ndarray) else x


def gram(pat, o):
    return int.from_bytes(bytes(pat[o:o + 4]), "little")


def qsample_count(pats, ks, buf, buf_lo, own_lo, own_hi, generic=False):
    """Distinct (pattern ordinal, granule) pairs k_filter_multi marks."""
    return sum(g.size for g in qsample_granules(pats, ks, buf, buf_lo, own_lo, own_hi, generic))


def qsample_granules(pats, ks, buf, buf_lo, own_lo, own_hi, generic=False):
    """Per pattern, the granules (buffer-relative, ascending) k_filter_multi marks."""
    buf = u8(buf)
    nw = (len(buf) + 15) // 16 * 4
    b = np.zeros(4 * nw, dtype=np.uint8)
    b[:len(buf)] = buf
    words = b.view("<u4")
    out = []
    for P, k in zip(pats, ks):
        m = len(P)
        L, K = m // (k + 1), (2 * k if generic else k)
        parts = []
        for o in range(m - 3):
            a = buf_lo + 4 * np.flatnonzero(words == gram(P, o)).astype(np.int64) - o
            lo, hi = np.maximum(a - K, own_lo), np.minimum(a + K + m - L, own_hi - 1)
            keep = lo <= hi
            g0, g1 = (lo[keep] - buf_lo) >> 6, (hi[keep] - buf_lo) >> 6
            for d in range(int((g1 - g0).max()) + 1 if g0.size else 0):
                parts.append((g0 + d)[g0 + d <= g1])
        out.append(np.unique(np.concatenate(parts)) if parts else np.zeros(0, dtype=np.int64))
    return out


def eq_run(buf, lo, hi, piece, code=None):
    """Boolean over the buffer positions g in [lo, hi): buf[g+q] equals piece[q] for every q (under `code`: their
    codes do).  Positions past the buffer read as zeros."""
    pad = np.zeros(hi + len(piece) - lo, dtype=np.uint8)
    src = buf[lo:hi + len(piece)]
    pad[:len(src)] = src
    eq = np.ones(max(hi - lo, 0), dtype=bool)
    for q, c in enumerate(piece):
        col = pad[q:q + hi - lo]
        eq &= (code[col] == code[c]) if code is not None else (col == c)
    return eq


def ngram_hits(pats, ks, buf, buf_lo, N, own_lo, own_hi):
    """Hits (pattern, n-gram j, g) of k_filter_mdense and k_filter_mdense2."""
    buf = u8(buf)
    total = 0
    for P, k in zip(pats, ks):
        P = u8(P)
        m = len(P)
        L = m // (k + 1)
        lo, hi = own_lo - buf_lo, min(own_hi, N - L + 1) - buf_lo
        assert hi + L - 1 <= len(buf) or hi <= lo, "the buffer must hold every n-gram that ends at or before N"
        for j in range(m // L):
            total += int(np.count_nonzero(eq_run(buf, lo, hi, P[j * L:(j + 1) * L])))
    return total


def two_bit_code(pats):
    """two_bit_code of api.cu: the four most frequent pattern bytes of the pass -> 0..3 (ties: the lower byte
    first), every other byte -> 0."""
    freq = np.zeros(256, dtype=np.int64)
    for P in pats:
        np.add.at(freq, u8(P), 1)
    order = sorted(range(256), key=lambda c: -freq[c])
    code = np.zeros(256, dtype=np.uint8)
    for r in range(4):
        code[order[r]] = r
    return code


def keys_at(buf, code=None):
    """The key at every buffer position: the 4 bytes there (little-endian), or the 2-bit codes of the 8 symbols there
    (symbol q at bits 2q, 2q+1); zeros past the end."""
    n = len(buf)
    width = 8 if code is not None else 4
    b = np.zeros(n + width, dtype=np.uint8)
    b[:n] = buf
    if code is not None:
        b = code[b]
    key = np.zeros(n, dtype=np.uint32)
    for q in range(width):
        key |= b[q:q + n].astype(np.uint32) << np.uint32(2 * q if code is not None else 8 * q)
    return key


def ham_key_hits(pats, ks, buf, buf_lo, N, own_lo, own_hi, two_bit=False):
    """(pattern, piece j, g) pairs k_ham_batch_scan counts as candidates."""
    buf = u8(buf)
    code = two_bit_code(pats) if two_bit else None
    keys = keys_at(buf, code)
    n = len(buf)
    total = 0
    for P, k in zip(pats, ks):
        P = u8(P)
        m = len(P)
        L = m // (k + 1)
        w = min(L, 8) if two_bit else min(L, 4)
        mask = (1 << ((2 if two_bit else 8) * w)) - 1
        for j in range(k + 1):
            want = int(keys_at(P[j * L:j * L + w], code)[0]) & mask
            lo = max(0, own_lo - buf_lo + j * L)
            hi = min(n, own_hi - buf_lo + j * L, N - m - buf_lo + j * L + 1)
            if hi > lo:
                total += int(np.count_nonzero((keys[lo:hi] & np.uint32(mask)) == want))
    return total


def lp_survivors(pats, ks, buf, buf_lo, N, own_lo, own_hi, generic=False):
    """Survivors (pattern, s) of k_lp_scan_multi."""
    buf = u8(buf)
    wmax = max(len(P) + k for P, k in zip(pats, ks))
    lim = min(N, buf_lo + len(buf)) - buf_lo
    s0, s1 = own_lo - buf_lo, min(own_hi - buf_lo, lim)
    if s1 <= s0:
        return 0
    total = 0
    for P, k in zip(pats, ks):
        P = u8(P)
        m = len(P)
        in_p = np.zeros(256, dtype=np.int32)
        in_p[P] = 1
        cs = np.zeros(lim + 1 + wmax, dtype=np.int32)  # cs[i]: bytes of P before min(i, lim)
        np.cumsum(in_p[buf[:lim]], out=cs[1:lim + 1])
        cs[lim + 1:] = cs[lim]
        ok = cs[s0 + wmax:s1 + wmax] - cs[s0:s1] >= m - k
        if not generic:
            first = np.zeros(256, dtype=bool)
            first[P[:min(k, m - 1) + 1]] = True
            ok &= first[buf[s0:s1]]
        total += int(np.count_nonzero(ok))
    return total


# ------------------------------------------------------------------------------------------------ the passes
class Pass(object):
    """One kind of shared pass: how to call it, the route its patterns report and its restatement."""

    def __init__(self, name, route, kind, count):
        self.name, self.route, self.kind, self.count = name, route, kind, count

    def batch(self, hs, pats, ks, flags=0):
        if self.kind == "ham":
            return hs.search_hamming_batch(pats, ks, flags)
        if self.kind == "generic":
            return hs.search_generic_batch(pats, ks, ks, ks, ks, flags=flags)
        return hs.search_levenshtein_batch(pats, ks, flags)

    def single(self, hs, pat, k):
        if self.kind == "ham":
            return hs.search_hamming(pat, k)
        if self.kind == "generic":
            return hs.search_generic(pat, k, k, k, k)
        return hs.search_levenshtein(pat, k)

    def oracle_raw(self, pat, hay, k):
        if self.kind == "ham":
            return oracle.substitutions(pat, hay, k)
        if self.kind == "generic":
            return oracle.generic_raw(pat, hay, k, k, k, k)
        return oracle.levenshtein_raw(pat, hay, k)

    def restate(self, pats, ks, buf, buf_lo=0, N=None, own_lo=None, own_hi=None):
        N = buf_lo + len(buf) if N is None else N
        own_lo = buf_lo if own_lo is None else own_lo
        own_hi = N if own_hi is None else own_hi
        return self.count(pats, ks, buf, buf_lo, N, own_lo, own_hi)


QSAMPLE = Pass("q-sample", SAMPLED, "lev", lambda p, k, b, lo, N, a, z: qsample_count(p, k, b, lo, a, z))
GQSAMPLE = Pass("generic q-sample", GSAMPLED, "generic",
                lambda p, k, b, lo, N, a, z: qsample_count(p, k, b, lo, a, z, generic=True))
PREFIX = Pass("prefix", DENSE, "lev", ngram_hits)
GPREFIX = Pass("generic prefix", GSAMPLED, "generic", ngram_hits)
TWO_BIT = Pass("2-bit", DENSE, "lev", ngram_hits)
HAM_TEXT = Pass("text keys", HAM, "ham", ham_key_hits)
HAM_2BIT = Pass("2-bit keys", HAM, "ham",
                lambda p, k, b, lo, N, a, z: ham_key_hits(p, k, b, lo, N, a, z, two_bit=True))
LPP = Pass("LP", LP, "lev", lp_survivors)
GLPP = Pass("generic LP", GLP, "generic",
            lambda p, k, b, lo, N, a, z: lp_survivors(p, k, b, lo, N, a, z, generic=True))


def run_pass(hs, ps, pats, ks, hay=None, flags=0, geom=None, want_launches=None, singles=None):
    """One batch call whose patterns all ride one pass of kind `ps`: the route of every result, the scan reported
    by the first pattern only, n_candidates against the restatement over `geom` = (buf, buf_lo, N, own_lo, own_hi),
    and every pattern's RAW (sorted) and FINAL against its single search on `hs` (only the patterns `singles`, if
    given) and, with `hay` (the whole sequence), the oracle.  -> (restated count, RAW records in all, n_launches of
    the pass)."""
    results, total = ps.batch(hs, pats, ks, flags)
    sts = [r.stats() for r in results]
    assert [s["route"] for s in sts] == [ps.route] * len(pats), (ps.name, sts)
    assert sts[0]["bytes_scanned"] > 0 and all(s["bytes_scanned"] == 0 for s in sts[1:]), (ps.name, sts)
    assert all(s["n_candidates"] == 0 and s["n_launches"] == 0 for s in sts[1:]), (ps.name, sts)
    if want_launches is not None:
        assert sts[0]["n_launches"] == want_launches, (ps.name, sts[0])
    want = ps.restate(pats, ks, *geom)
    assert sts[0]["n_candidates"] == total["n_candidates"] == want, (ps.name, sts[0]["n_candidates"], want)
    nraw = 0
    for q, (p, k, r) in enumerate(zip(pats, ks, results)):
        raw = sorted(r.triples(F.RAW))
        if singles is None or q in singles:
            one = ps.single(hs, p, k)
            assert raw == sorted(one.triples(F.RAW)), (ps.name, q)
            assert r.triples(F.FINAL) == one.triples(F.FINAL), (ps.name, q)
            one.close()
        if hay is not None and len(hay) <= ORACLE_MAX:
            assert raw == sorted(tup(ps.oracle_raw(p, bytes(hay), k))), (ps.name, q)
        nraw += len(raw)
        r.close()
    return want, nraw, sts[0]["n_launches"]


# ------------------------------------------------------------------------------------------------ contents
def rand(rng, alphabet, n):
    alpha = np.frombuffer(alphabet, dtype=np.uint8)
    return alpha[rng.integers(0, len(alpha), size=n)].copy()


def put(hay, pos, v):
    v = u8(v)[:max(0, len(hay) - pos)]
    if pos >= 0:
        hay[pos:pos + len(v)] = v


def plant_seams(rng, hay, pieces, seams, back=12):
    """At every seam b one of `pieces` starting 1 to `back` bytes before it: across a lane-31 vector seam, a warp
    seam or a tile seam (its first bytes in one vector, the rest in the next)."""
    for b in seams:
        pc = pieces[int(rng.integers(0, len(pieces)))]
        put(hay, b - int(rng.integers(1, back + 1)), pc)


def plantable(pats, ks):
    """The patterns a test plants: not those with k = 8 (the LP pass's wmax = 31), whose occurrences leave a start
    with more live automaton candidates than the LP pass's verification lists hold -- the pass then goes one by one.
    Unplanted, such a pattern still sets wmax and is counted wherever random text survives."""
    keep = [q for q, k in enumerate(ks) if k < 8]
    return [pats[q] for q in keep], [ks[q] for q in keep]


def plant_copies(rng, hay, pats, ks, alphabet, every, subs_only=False):
    pats, ks = plantable(pats, ks)
    for s in range(int(rng.integers(0, every)), len(hay) - 80, every):
        q = int(rng.integers(0, len(pats)))
        p, k = pats[q], ks[q]
        e = int(rng.integers(0, k + 2))
        if subs_only:
            v = bytearray(p)
            for i in rng.choice(len(v), size=min(e, len(v)), replace=False):
                v[i] = alphabet[int(rng.integers(0, len(alphabet)))]
            put(hay, s, bytes(v))
        else:
            put(hay, s, mutate(rng, p, alphabet, e))


def seams_of(n, small):
    """lane-31 vector seams of the first and last warps, warp seams, tile seams and the last vector"""
    seams = set(range(16 * 31 + 16, min(n, 8 * WARP), WARP))
    seams |= set(range(WARP, n, WARP if small else 61 * WARP))
    seams |= set(range(TILE, n, TILE)) | {max(16, (n - 1) // 16 * 16)}
    return sorted(s for s in seams if 16 <= s < n)


def lengths_around(tiles, grid):
    """every residue mod 16 around one and two tiles; around one, two (plus one) and three passes of the grid"""
    out = [b + d for b in (tiles, 2 * tiles) for d in range(-8, 8)]
    return out + [grid * tiles + 1, (2 * grid + 1) * tiles + 3, 3 * grid * tiles - 5]


# ------------------------------------------------------------------------------------------------ the mixes
def qsample_mix(rng):
    """q-sample lemma holds (m - k - 3) // 4 >= k + 1; a duplicate, a periodic pattern"""
    pats = [bytes(rand(rng, ASCII, m)) for m in (24, 32, 40, 64)]
    pats += [pats[1], b"abcdefgh" * 4]
    return pats, [1, 2, 3, 4, 1, 2]


def prefix_mix(rng):
    """n-gram route patterns the lemma does not cover: L = m // (k + 1) from 3 to 5, a duplicate, repeated n-grams"""
    pats = [bytes(rand(rng, ASCII, m)) for m in (10, 12, 9, 11, 20)]
    pats += [pats[0], b"xyz" * 4]
    return pats, [2, 2, 1, 1, 5, 2, 3]


def dna_mix(rng):
    """2-bit pass: n-grams of 5, 7, 8 and 10 symbols, a duplicate, a byte outside the four codes"""
    pats = [bytes(rand(rng, DNA, m)) for m in (15, 21, 16, 20)]
    pats += [pats[0], bytes(rand(rng, DNA, 9)) + b"N" + bytes(rand(rng, DNA, 10))]
    return pats, [2, 2, 1, 1, 2, 1]


def lp_mix(rng):
    """LP route, m // (k + 1) < 3: need = m - k from 1 (m 2, k 1) to 15, wmax = m + k = 31 (m 23, k 8)"""
    pats = [bytes(rand(rng, ASCII, m)) for m in (5, 8, 2, 23, 12)]
    return pats, [2, 3, 1, 8, 4]


def ham_text_mix(rng):
    pats = [bytes(rand(rng, ASCII, m)) for m in (20, 16, 33, 64)]
    return pats + [pats[0]], [3, 1, 2, 7, 2]


def ham_2bit_mix(rng):
    pats = [bytes(rand(rng, DNA, m)) for m in (20, 24, 32, 40)]
    return pats + [pats[1][:12] + b"N" + pats[1][13:]], [3, 2, 1, 4, 2]


def pieces_of(pats, ks, L=None):
    pats, ks = plantable(pats, ks)
    out = []
    for p, k in zip(pats, ks):
        ln = L or len(p) // (k + 1)
        out += [p[j * ln:(j + 1) * ln] for j in range(len(p) // ln)]
    return out


# ------------------------------------------------------------------------------------------------ tests
def lengths_case(ps, mix, alphabet, tile, grid, small, subs_only=False, seed=0):
    rng = np.random.default_rng(seed)
    pats, ks = mix(rng)
    lengths = lengths_around(tile, grid)
    base = rand(rng, alphabet, max(lengths) + 64)
    plant_seams(rng, base, pieces_of(pats, ks) + [p[:4] for p in pats], seams_of(len(base), small))
    plant_copies(rng, base, pats, ks, alphabet, 997 if small else 9973, subs_only)
    cands = raw = 0
    for n in lengths:
        hay = base[:n].copy()
        put(hay, 0, pats[0])
        put(hay, n - len(pats[-1]), pats[-1])
        hs = F.Haystack.from_host(hay)
        # (past two tiles the lists of the first and the last pattern stand for the rest: the single searches of
        # every pattern over three grid passes would take most of a minute)
        c, r, _ = run_pass(hs, ps, pats, ks, hay=hay, geom=(hay,), singles=None if n < 3 * tile else (0, len(pats) - 1))
        cands, raw = cands + c, raw + r
        hs.close()
    assert cands > len(lengths) and raw >= len(lengths)


def test_qsample_lengths(cuda_device, small=False):
    lengths_case(QSAMPLE, qsample_mix, ASCII, TILE, EMU_SMS if small else SMS, small, seed=601)


def test_prefix_lengths(cuda_device, small=False):
    lengths_case(PREFIX, prefix_mix, ASCII, TILE, EMU_SMS if small else SMS, small, seed=602)


def test_two_bit_lengths(cuda_device, small=False):
    lengths_case(TWO_BIT, dna_mix, DNA, TILE, EMU_SMS if small else SMS, small, seed=603)


def test_ham_lengths(cuda_device, small=False):
    sms = EMU_SMS if small else SMS
    lengths_case(HAM_TEXT, ham_text_mix, ASCII, TILE, sms, small, subs_only=True, seed=604)
    lengths_case(HAM_2BIT, ham_2bit_mix, DNA, TILE, 2 * sms, small, subs_only=True, seed=605)


def test_lp_lengths(cuda_device, small=False):
    lengths_case(LPP, lp_mix, ASCII, LP_TILE, 2 * (EMU_SMS if small else SMS), small, seed=606)


def test_generic_passes(cuda_device, small=False):
    """Generic patterns: the q-sample pass marks around 2k, the prefix pass finds the same hits, the LP pass takes
    every first byte."""
    rng = np.random.default_rng(607)
    n = 2 * TILE + 333 if small else 5 * TILE + 333
    for ps, pats, ks in ((GQSAMPLE, [bytes(rand(rng, ASCII, m)) for m in (24, 40, 33)], [1, 2, 2]),
                         (GPREFIX, [bytes(rand(rng, ASCII, m)) for m in (10, 12, 16)], [2, 2, 1]),
                         (GLPP, [bytes(rand(rng, ASCII, m)) for m in (5, 9, 12)], [2, 3, 4])):
        hay = rand(rng, ASCII, n)
        plant_seams(rng, hay, pieces_of(pats, ks) + [p[:4] for p in pats], seams_of(n, small))
        plant_copies(rng, hay, pats, ks, ASCII, 1999)
        hs = F.Haystack.from_host(hay)
        c, r, _ = run_pass(hs, ps, pats, ks, hay=hay if small else None, geom=(hay,))
        assert c > 0 and r > 0, ps.name
        hs.close()


def test_nul_grams_and_reupload(cuda_device, small=False):
    """Patterns holding NULs against the zero padding behind the buffer (the last vector's words, the prefix and key
    bytes past the end), then shorter contents uploaded over a buffer full of occurrences: stale bytes past the new
    end would add candidates."""
    rng = np.random.default_rng(608)
    cases = [(QSAMPLE, [b"\0" * 8 + bytes(rand(rng, ASCII, 24)), bytes(rand(rng, ASCII, 28)) + b"\0" * 4], [1, 2]),
             (PREFIX, [bytes(rand(rng, ASCII, 9)) + b"\0\0\0", b"\0" * 4 + bytes(rand(rng, ASCII, 8))], [2, 2]),
             (HAM_TEXT, [bytes(rand(rng, ASCII, 12)) + b"\0" * 8, b"\0\0\0" + bytes(rand(rng, ASCII, 13))], [3, 3]),
             (LPP, [b"\0a\0b\0", bytes(rand(rng, ASCII, 6)) + b"\0"], [2, 3])]
    for ps, pats, ks in cases:
        n0 = 2 * TILE + 100
        full = np.frombuffer(b"".join(pats) * (n0 // sum(map(len, pats)) + 1), dtype=np.uint8)[:n0].copy()
        hs = F.Haystack.from_host(full)
        run_pass(hs, ps, pats, ks, geom=(full,))
        for n in [TILE + d for d in (-9, -1, 0, 3, 7)] + [1000 + d for d in range(16)]:
            hay = rand(rng, ASCII, n)
            hay[-int(rng.integers(1, 14)):] = 0
            put(hay, n - len(pats[0]) + 3, pats[0])
            put(hay, 100, pats[1])
            hs.upload(hay)
            run_pass(hs, ps, pats, ks, hay=hay, geom=(hay,))
        hs.close()


def test_packed_tiles(cuda_device, small=False):
    """One CTA's tile holding more entries than its buffer: past the flush threshold (1 024 hits of the n-gram
    passes, 2 048 LP survivors), past the capacity (3 072, 6 144) into the straight-to-global path; and keys with more
    than 255 postings, which spill over several table slots."""
    rng = np.random.default_rng(609)
    # n-gram passes: one tile packed with copies of two patterns (every n-gram of every copy is a hit)
    for ps, alphabet, pats, ks in ((PREFIX, ASCII, [bytes(rand(rng, ASCII, 12)), bytes(rand(rng, ASCII, 10))], [2, 2]),
                                   (TWO_BIT, DNA, [bytes(rand(rng, DNA, 15)), bytes(rand(rng, DNA, 20))], [2, 1])):
        n = 3 * TILE + 77
        hay = rand(rng, alphabet, n)
        run = (pats[0] * 1500 + pats[1] * 1500)[:TILE - 500]
        put(hay, TILE + 100, run)
        hs = F.Haystack.from_host(hay)
        c, _, _ = run_pass(hs, ps, pats, ks, hay=hay if small else None, geom=(hay,))
        assert c > 6144, (ps.name, c)
        hs.close()
    # LP: a tile of text made of the patterns' bytes: nearly every start survives for every pattern
    pats = [b"abcde", b"bcdea", b"cdeab", b"aabbc"]
    ks = [2, 2, 3, 2]
    n = 3 * LP_TILE + 99
    hay = rand(rng, ASCII, n)
    put(hay, LP_TILE + 64, rand(rng, b"abcde", LP_TILE))
    hs = F.Haystack.from_host(hay)
    c, _, _ = run_pass(hs, LPP, pats, ks, hay=hay if small else None, geom=(hay,))
    assert c > 6144 * 2
    hs.close()
    # postings: 300 patterns sharing their first gram, prefix and key (q-sample, prefix, Hamming text keys)
    n = TILE + 4321
    for ps, m, k in ((QSAMPLE, 24, 1), (PREFIX, 12, 2), (HAM_TEXT, 16, 3)):
        head = bytes(rand(rng, ASCII, 4))
        pats = [head + bytes(rand(rng, ASCII, m - 4)) for _ in range(300)]
        ks = [k] * len(pats)
        hay = rand(rng, ASCII, n)
        for s in range(50, n - 100, 997 if small else 331):
            put(hay, s, pats[int(rng.integers(0, len(pats)))] if rng.random() < 0.5 else head)
        hs = F.Haystack.from_host(hay)
        results, _ = ps.batch(hs, pats, ks)
        sts = [r.stats() for r in results]
        assert [s["route"] for s in sts] == [ps.route] * len(pats) and sum(s["bytes_scanned"] > 0 for s in sts) == 1
        got = sum(s["n_candidates"] for s in sts)
        assert got == ps.restate(pats, ks, hay) > 0, ps.name
        for q in rng.choice(len(pats), size=6, replace=False):
            one = ps.single(hs, pats[q], k)
            assert sorted(results[q].triples(F.RAW)) == sorted(one.triples(F.RAW)), (ps.name, q)
            one.close()
        for r in results:
            r.close()
        hs.close()


def level1_colliders(rng, w, count, bits=20):
    """`count` u32 words whose level-1 hash (w * kHashMul) >> (32 - bits) equals w's, none equal to w."""
    h = ((w * HASH) & 0xFFFFFFFF) >> (32 - bits)
    top = (h << (32 - bits)) | rng.integers(0, 1 << (32 - bits), size=count, dtype=np.uint64)
    out = ((top * np.uint64(HASH_INV)) & np.uint64(0xFFFFFFFF)).astype(np.uint32)
    return out[out != w]


def test_hash_collisions(cuda_device, small=False):
    """Words in the level-1 bucket of a pattern gram (q-sample) or text key (Hamming) without equalling it, at
    aligned words and at every byte offset: the postings table compares exactly, so they add nothing."""
    rng = np.random.default_rng(610)
    n = 2 * TILE + 555 if small else 4 * TILE + 555
    for ps, pats, ks in ((QSAMPLE, [bytes(rand(rng, ASCII, m)) for m in (24, 32)], [1, 2]),
                         (HAM_TEXT, [bytes(rand(rng, ASCII, m)) for m in (20, 16)], [3, 1])):
        hay = rand(rng, ASCII, n)
        grams = [gram(p, o) for p in pats for o in range(len(p) - 3)] if ps is QSAMPLE else \
            [gram(p, j * (len(p) // (k + 1))) for p, k in zip(pats, ks) for j in range(k + 1)]
        col = np.concatenate([level1_colliders(rng, g, 40) for g in grams])
        pos = rng.choice(np.arange(0, n - 8, 4 if ps is QSAMPLE else 1), size=min(col.size, n // 16), replace=False)
        for p, w in zip(pos, col):
            put(hay, int(p), int(w).to_bytes(4, "little"))
        plant_copies(rng, hay, pats, ks, ASCII, 2999, subs_only=ps is HAM_TEXT)
        hs = F.Haystack.from_host(hay)
        c, r, _ = run_pass(hs, ps, pats, ks, hay=hay if small else None, geom=(hay,))
        assert c > 0 and r > 0
        hs.close()


def test_shards(cuda_device, small=False):
    """Shards whose buffers start at buf_lo != 0 (a multiple of 16 off the 64 KiB tiles and 128-byte runs), then at
    40- and 44-bit offsets: each count is the restatement of the shard's own buffer and range."""
    rng = np.random.default_rng(611)
    n = 3 * TILE + 4321 if small else 6 * TILE + 4321
    for ps, mix, alphabet in ((QSAMPLE, qsample_mix, ASCII), (PREFIX, prefix_mix, ASCII), (TWO_BIT, dna_mix, DNA),
                              (HAM_TEXT, ham_text_mix, ASCII), (LPP, lp_mix, ASCII)):
        pats, ks = mix(rng)
        m = max(map(len, pats)) + max(ks)
        hay = rand(rng, alphabet, n)
        plant_copies(rng, hay, pats, ks, alphabet, 1499, subs_only=ps is HAM_TEXT)
        bounds = [0, n // 3 + 5, 2 * n // 3 - 7, n]
        plant_seams(rng, hay, pieces_of(pats, ks), bounds[1:-1] + seams_of(n, True))
        for i in range(3):
            lo, hi = bounds[i], bounds[i + 1]
            blo = max(0, lo - m) // 16 * 16
            if blo % 128 == 0 and blo > 0:
                blo -= 16
            bhi = min(n, hi + m)
            hs = F.Haystack.from_host(hay[blo:bhi], buf_lo=blo, global_len=n, own_lo=lo, own_hi=hi)
            results, _ = ps.batch(hs, pats, ks)
            sts = [r.stats() for r in results]
            assert [s["route"] for s in sts] == [ps.route] * len(pats), (ps.name, i)
            assert sum(s["bytes_scanned"] > 0 for s in sts) == 1, (ps.name, i)
            got = sum(s["n_candidates"] for s in sts)
            assert got == ps.restate(pats, ks, hay[blo:bhi], blo, n, lo, hi), (ps.name, i)
            for r in results:
                r.close()
            hs.close()
        for shift in ((1 << 40) + 16 * 12345, 1 << 44):
            G = shift + n + (1 << 20)
            hs = F.Haystack.from_host(hay, buf_lo=shift, global_len=G, own_lo=shift + 256, own_hi=shift + n - m)
            results, _ = ps.batch(hs, pats, ks)
            assert [r.stats()["route"] for r in results] == [ps.route] * len(pats), (ps.name, shift)
            assert sum(r.stats()["bytes_scanned"] > 0 for r in results) == 1, (ps.name, shift)
            got = sum(r.stats()["n_candidates"] for r in results)
            assert got == ps.restate(pats, ks, hay, shift, G, shift + 256, shift + n - m) > 0, (ps.name, shift)
            for q in (0, len(pats) - 1):
                one = ps.single(hs, pats[q], ks[q])
                assert sorted(results[q].triples(F.RAW)) == sorted(one.triples(F.RAW)), (ps.name, shift, q)
                one.close()
            for r in results:
                r.close()
            hs.close()


def test_record_sets(cuda_device, small=False):
    """Record sets: the filters read content only, so with FZB_F_PER_RECORD the count of each pass is the restatement
    over the joined buffer, separators included; fzb_best_per_record runs the same passes and reports the same sum."""
    rng = np.random.default_rng(612)
    for ps, mix, alphabet in ((QSAMPLE, qsample_mix, ASCII), (PREFIX, prefix_mix, ASCII), (TWO_BIT, dna_mix, DNA),
                              (HAM_TEXT, ham_text_mix, ASCII), (LPP, lp_mix, ASCII)):
        pats, ks = mix(rng)
        recs = []
        total = 0
        while total < (TILE + 999 if small else 3 * TILE + 999):
            r = bytearray(rand(rng, alphabet, int(rng.integers(0, 400))))
            if len(r) > 80 and rng.random() < 0.7:
                pp = plantable(pats, ks)[0]
                p = pp[int(rng.integers(0, len(pp)))]
                pos = int(rng.integers(0, len(r) - len(p)))
                r[pos:pos + len(p)] = p
            recs.append(bytes(r))
            total += len(r) + 1
        buf = np.frombuffer(b"\0".join(recs) + b"\0", dtype=np.uint8)
        off = np.zeros(len(recs) + 1, dtype=np.uint64)
        off[1:] = np.cumsum([len(r) + 1 for r in recs])
        hs = F.Haystack.from_host(buf)
        hs.set_records(off)
        want = ps.restate(pats, ks, buf)
        results, tot = ps.batch(hs, pats, ks, F.F_PER_RECORD)
        sts = [r.stats() for r in results]
        assert [s["route"] for s in sts] == [ps.route] * len(pats), ps.name
        assert sum(s["bytes_scanned"] > 0 for s in sts) == 1, ps.name
        assert sum(s["n_candidates"] for s in sts) == tot["n_candidates"] == want > 0, ps.name
        for q, (p, k, r) in enumerate(zip(pats, ks, results)):
            one = ps.single(hs, p, k)
            assert sorted(r.triples(F.RAW)) == sorted(one.triples(F.RAW)), (ps.name, q)
            assert r.triples(F.FINAL) == one.triples(F.FINAL), (ps.name, q)
            one.close()
            r.close()
        if ps.kind == "ham":
            _, st = hs.best_per_record(pats, ks, [0] * len(ks), [0] * len(ks), ks)
        else:
            _, st = hs.best_per_record(pats, ks, ks, ks, ks)
        assert st["n_candidates"] == want, ps.name
        hs.close()


def test_tiny_chunks(cuda_device, small=False):
    """FZB_F_TINY_LIST: the 2-bit and LP passes scan chunks of 3 000 positions (seams inside a vector, a 128-byte run
    and a tile) with small lists; on sparse contents that stay under those caps the count is the same with and
    without the flag, and the 2-bit pass reports two launches per chunk, the LP pass four."""
    rng = np.random.default_rng(613)
    n = 7 * TINY_CHUNK + 123 if small else 25 * TINY_CHUNK + 123
    # 2-bit: n-grams of 10 symbols and more, at most 6 hits per chunk, straddling every seam
    pats = [bytes(rand(rng, DNA, m)) for m in (20, 24, 30, 40)]
    ks = [1, 1, 1, 1]
    hay = rand(rng, DNA, n)
    for c in range(1, n // TINY_CHUNK + 1):
        seam = c * TINY_CHUNK
        p = pats[c % 4]
        put(hay, seam - len(p) // 2 - int(rng.integers(0, 3)), p)
    hs = F.Haystack.from_host(hay)
    chunks = (n + TINY_CHUNK - 1) // TINY_CHUNK
    a, _, _ = run_pass(hs, TWO_BIT, pats, ks, hay=hay, flags=F.F_TINY_LIST, geom=(hay,), want_launches=2 * chunks)
    b, _, _ = run_pass(hs, TWO_BIT, pats, ks, hay=hay, geom=(hay,), want_launches=2)
    assert a == b > 0
    hs.close()
    # LP: text whose windows rarely reach need, survivors planted across every chunk seam
    pats, ks = [b"qrstuvwx", b"QRSTU"], [3, 2]
    hay = rand(rng, b"abcdefghijklmnopABCDEFGHIJ0123456789", n)
    for c in range(1, n // TINY_CHUNK + 1):
        put(hay, c * TINY_CHUNK - 4 + int(rng.integers(0, 3)), pats[c % 2])
    put(hay, n - 5, pats[1])
    hs = F.Haystack.from_host(hay)
    a, _, _ = run_pass(hs, LPP, pats, ks, hay=hay, flags=F.F_TINY_LIST, geom=(hay,), want_launches=4 * chunks)
    b, _, _ = run_pass(hs, LPP, pats, ks, hay=hay, geom=(hay,), want_launches=4)
    assert a == b > 0
    hs.close()
