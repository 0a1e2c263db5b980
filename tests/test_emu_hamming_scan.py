"""The tile, ring and counter geometry of k_hamming_count replayed on the emulated build: the bodies of the -m gpu
tests of test_gpu_hamming_scan.py, with one pass of the emulated grid (4 CTAs) in place of the H100's.

Before that, the restatement those tests compare with is checked on its own, without a device: it covers every
true match (brute force), and it equals a literal transcription of the kernel's per-row loop (ham_sliced_step and
ham_sliced2_step of ham_recur.h, 7 warm-up words from the previous row, the carries of the row's own 32 words
or-ed into `acc`).  A mismatch on the device then points at the device."""
import numpy as np

import test_gpu_hamming_scan as G
from test_emu_kernels import emu_device, emu_lib  # noqa: F401  (fixtures)

M32 = 0xFFFFFFFF


def ham_sliced_step(s, M, B0, B1, B2):
    x0 = ((s[0] + s[0]) & 0xFEFEFEFE) | B0
    x1 = ((s[1] + s[1]) & 0xFEFEFEFE) | B1
    x2 = ((s[2] + s[2]) & 0xFEFEFEFE) | B2
    c0 = x0 & M
    s[0] = x0 ^ M
    c1 = x1 & c0
    s[1] = x1 ^ c0
    s[2] = x2 ^ c1
    return x2 & c1


def ham_sliced2_step(s, M, B0, B1):
    x0 = ((s[0] + s[0]) & 0xFEFEFEFE) | B0
    x1 = ((s[1] + s[1]) & 0xFEFEFEFE) | B1
    c0 = x0 & M
    s[0] = x0 ^ M
    s[1] = x1 ^ c0
    return x1 & c0


def kernel_rows(pat, k, buf, slices=None):
    """The rows k_hamming_count flags, one row at a time as its threads run them."""
    Wc, _, S, bias = G.layout(len(pat), k, slices)
    table = [0] * 256
    for o0 in range(4):
        for i in range(Wc):
            table[int(G.bucket(G.gram(pat, o0 + 4 * i)))] |= 1 << (8 * o0 + i)
    B = [0x01010101 if (bias >> j) & 1 else 0 for j in range(3)]
    words = [int(w) for w in G.scanned_words(buf)]
    rows = []
    for r in range(len(words) // 32):
        s = [0, 0, 0]
        acc = 0
        for t in range(32 * r - 7, 32 * r + 32):  # 7 warm-up words, then the row's own
            M = table[int(G.bucket(words[t] if t >= 0 else 0))]
            c = ham_sliced2_step(s, M, B[0], B[1]) if S == 2 else ham_sliced_step(s, M, B[0], B[1], B[2])
            if t >= 32 * r:
                acc |= c & M32
        if acc:
            rows.append(r)
    return rows


def planted(rng, alphabet, n, m, k):
    pat = bytes(G.random_text(rng, m, alphabet))
    hay = G.random_text(rng, n, alphabet)
    for t in range(40):
        pos = 0 if t == 0 else n - m if t == 1 else int(rng.integers(0, n - m + 1))
        G.put(hay, pos, G.subs(rng, pat, int(rng.integers(0, k + 2))))
    return pat, hay


def test_restatement_covers_every_match():
    """Every start p with Hamming(P, H[p:p+m]) <= k lies in a marked range, with the host's slice choice and, where
    the threshold allows two slices, with three: over random texts of the alphabets of ham_recur_check.cpp."""
    rng = np.random.default_rng(31)
    checked = 0
    for trial in range(90):
        alphabet = (b"ACGT", b"ab", b"abcdefghijklmnopqrstuvwxyz")[trial % 3]
        k = int(rng.integers(0, 8))
        m = 4 * k + 7 + int(rng.integers(0, 40)) + (60 if trial % 5 == 0 else 0)
        n = int(rng.integers(m, 6000))
        pat, hay = planted(rng, alphabet, n, m, k)
        windows = np.lib.stride_tricks.sliding_window_view(hay, m)
        starts = np.nonzero((windows != np.frombuffer(pat, dtype=np.uint8)).sum(axis=1) <= k)[0]
        assert starts.size > 0
        checked += starts.size
        T = G.layout(m, k)[1]
        for slices in (None, 3) if T <= 4 else (None,):
            lo, hi = G.mark_ranges(pat, k, hay, 0, 0, n, slices)
            covered = np.zeros(n + 1, dtype=np.int64)
            np.add.at(covered, lo, 1)
            np.add.at(covered, hi + 1, -1)
            assert (np.cumsum(covered)[starts] > 0).all(), (trial, m, k, slices)
    assert checked > 1000


def test_restatement_equals_the_kernel_loop():
    """The vectorised restatement flags the rows a literal transcription of the kernel's loop flags: every layout
    of test_counter_layouts, both slice counts where both apply, texts that end inside a row and hold NULs."""
    rng = np.random.default_rng(32)
    for i, (m, k) in enumerate(G.LAYOUTS):
        alphabet = (b"ab", b"ACGT", b"ab\0", G.ASCII)[i % 4]
        n = int(rng.integers(m, 3000))
        pat, hay = planted(rng, alphabet, n, m, k)
        T = G.layout(m, k)[1]
        for slices in (None, 3) if T <= 4 else (None,):
            want = kernel_rows(pat, k, hay, slices)
            assert G.flagged_rows(pat, k, hay, slices).tolist() == want, (m, k, slices)
    pat = b"\0" * 20 + b"0123456789ab"
    hay = np.zeros(300, dtype=np.uint8)
    assert G.flagged_rows(pat, 3, hay).tolist() == kernel_rows(pat, 3, hay) != []


def test_two_slice_double_carries_change_the_marks():
    """The counted words placed by carry_plants make two slices flag, at every plant, the row after the one both
    layouts flag, at every threshold from 1 to 4; where two slices carry once they mark what three slices mark."""
    rng = np.random.default_rng(33)
    rows = [3, 9, 15]
    for m, k in G.LAYOUTS:
        if G.layout(m, k)[2] != 2:
            continue
        pat = G.distinct_grams_pattern(rng, m, k)
        hay = G.quiet_text(rng, 3000, pat, k)
        G.carry_plants(hay, pat, k, rows)
        two = G.flagged_rows(pat, k, hay).tolist()
        three = G.flagged_rows(pat, k, hay, slices=3).tolist()
        assert three == rows, (m, k)
        assert two == (sorted(rows + [r + 1 for r in rows]) if G.double_carry(m, k) else rows), (m, k)
        if G.double_carry(m, k):
            assert len(G.hamming_marks(pat, k, hay, 0, 0, 3000)) > len(G.hamming_marks(pat, k, hay, 0, 0, 3000, 3))


def test_emu_hamming_scan_lengths(emu_device):
    G.test_buffer_lengths_around_tiles_and_grid_passes(emu_device, small=True)


def test_emu_hamming_scan_counters(emu_device):
    G.test_counter_layouts(emu_device, small=True)
    for k in range(8):
        G.test_dispatch_boundary(emu_device, k, small=True)
    G.test_hash_collisions(emu_device, small=True)


def test_emu_hamming_scan_edges(emu_device):
    G.test_nul_grams_against_the_zeros(emu_device, small=True)
    G.test_shards(emu_device, small=True)
    G.test_tiny_work_list_overflows_into_bitmap_mode(emu_device, small=True)
    G.test_record_sets(emu_device, small=True)
    G.test_reupload_shorter_contents(emu_device, small=True)
