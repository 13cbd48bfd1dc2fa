"""The row-driven kernels (row_kernels.cu) against the oracle, bit for bit, where they can go wrong.

A warp walks a row in 2 KiB staging segments: the first holds 2048 - off bytes (off = the address of the row's first
byte mod 16), and each later one starts span - 1 bytes before the previous one ends (span = k, or the minimizer window
in bases).  The inputs here put row lengths at -1, 0 and +1 around the first three segment edges, for every address
mod 16 and with the view itself at every byte offset from an aligned allocation.  Every byte of the allocation that no
row covers is poison ('N', or code 7 for byte codes), so a kernel that reads past a row changes a value or reports a
bad base.  The segment rule is restated here only to place the lengths; the oracle decides what is correct.

Every entry point of the C-ABI that takes a ragged view runs in every encoding (ACGT and ACTG text with lower case,
byte codes, a LUT with the ACGT, ACTG and ATCG tables): encode, k-mer hash, canonical hash, minimizers (both window
paths), the hashed count in every table mode, the exact table with growth, the generic-alphabet hash, the reverse
complement and the bincounts.  Bad bytes sit in segment overlaps, right after them and on the last byte of a row
that ends on a segment edge.  The long-row split of the Python layer is checked on CPU tensors and end to end."""
import functools
import os
import re
import shutil
import subprocess
from collections import namedtuple

import numpy as np
import pytest
import torch

from bionumpy_b200 import _native as nv
from oracle import bnp_oracle as o

gpu = pytest.mark.gpu

SEG = 2048                                        # bytes a warp stages per segment (kSegBytes)
INT64_MAX = (1 << 63) - 1
AMINO = "ACDEFGHIKLMNPQRSTVWY"
TEXT = np.frombuffer(b"ACGTacgt", dtype=np.uint8)

# mode / lut: what the kernel is given; table: the oracle's byte -> code table (255 = invalid); alphabet: the letter
# order of the codes (decides the complement)
Enc = namedtuple("Enc", "mode lut table size letters poison alphabet")


def _codes_table():
    t = np.full(256, 255, dtype=np.uint8)
    t[:4] = np.arange(4)
    return t


def _text(mode, alphabet, lut=False):
    table = o.alphabet_lut(alphabet)
    return Enc(mode, table if lut else None, table, 4, TEXT, ord("N"), alphabet)


ENCODINGS = {
    "acgt": _text(nv.ENC_ASCII_ACGT, "ACGT"),
    "actg": _text(nv.ENC_ASCII_ACTG, "ACTG"),
    "codes": Enc(nv.ENC_CODES, None, _codes_table(), 4, np.arange(4, dtype=np.uint8), 7, "ACGT"),
    "lut_acgt": _text(nv.ENC_LUT, "ACGT", lut=True),
    "lut_actg": _text(nv.ENC_LUT, "ACTG", lut=True),
    "lut_atcg": _text(nv.ENC_LUT, "ATCG", lut=True),
}
ENC_NAMES = list(ENCODINGS)
AMINO_ENC = Enc(nv.ENC_LUT, o.alphabet_lut(AMINO), o.alphabet_lut(AMINO), 20,
                np.frombuffer((AMINO + AMINO.lower()).encode(), dtype=np.uint8), ord("X"), AMINO)
CX_ALPHABET = {1: "ATCG", 2: "ACTG", 3: "ACGT"}          # the complement as an XOR on the 2-bit code
CX_OF = {a: cx for cx, a in CX_ALPHABET.items()}
# (encoding, complement_xor): every text encoding with its own alphabet, byte codes with all three
CANONICAL = [(e, CX_OF[ENCODINGS[e].alphabet]) for e in ENC_NAMES if e != "codes"] + [("codes", cx) for cx in (1, 2, 3)]


def segment_edges(off0, span, n=3):
    """Row lengths that fill the first n segments exactly, for a row whose first byte is at address off0 mod 16."""
    edges, start = [], 0
    for _ in range(n):
        end = start + SEG - (off0 + start) % 16
        edges.append(end)
        start = end - (span - 1)
    return edges


class Ragged:
    """Views into one aligned device allocation, each with its own rows (start relative to the view, length).  Bytes
    covered by a row are random letters of the encoding, every other byte of the allocation is poison."""

    def __init__(self, enc, views, view_rows, rng, bad=()):
        self.enc = enc
        size = max(vs + n for vs, n in views) + 64
        cover = np.zeros(size, dtype=bool)
        for (vs, _), rows in zip(views, view_rows):
            for s, L in rows:
                cover[vs + s: vs + s + L] = True
        self.host = np.where(cover, rng.choice(enc.letters, size=size), np.uint8(enc.poison)).astype(np.uint8)
        for view, row, pos in bad:                     # (view, row, position in row) -> poison
            s, L = view_rows[view][row]
            assert 0 <= pos < L
            self.host[views[view][0] + s + pos] = enc.poison
        self.views, self.view_rows = views, view_rows
        self.starts = np.array([s for rows in view_rows for s, _ in rows], dtype=np.int64)
        self.lens = np.array([L for rows in view_rows for _, L in rows], dtype=np.int32)
        abs_starts = np.array([vs + s for (vs, _), rows in zip(views, view_rows) for s, _ in rows], dtype=np.int64)
        self.flat = o.gather_rows(self.host, abs_starts, self.lens)
        first = np.cumsum([0] + [len(r) for r in view_rows])
        self.slices = [(int(first[i]), len(r)) for i, r in enumerate(view_rows)]
        self.alloc = torch.from_numpy(self.host).cuda()
        assert self.alloc.data_ptr() % 16 == 0
        self.bases = [self.alloc[vs: vs + n] for vs, n in views]
        self.d_starts = torch.from_numpy(self.starts).cuda()
        self.d_lens = torch.from_numpy(self.lens).cuda()
        self.lut = None if enc.lut is None else torch.from_numpy(enc.lut).cuda()

    @functools.cached_property
    def codes(self):
        return o.encode_flat(self.flat, self.enc.table, self.enc.size)

    def run(self, fn, params, shrink=None, dtype=torch.int64):
        """fn(base, n, starts, lens, n_rows, enc_mode, lut, *params[, offsets, out], status, stream), once per view.
        With ``shrink``, the views write one output (row r: max(len - shrink, 0) values).  Returns (out, statuses)."""
        out = off = None
        if shrink is not None:
            n = np.maximum(self.lens.astype(np.int64) - shrink, 0)
            off = torch.from_numpy(np.cumsum(n) - n).cuda()
            out = torch.empty(int(n.sum()), dtype=dtype, device="cuda")
        status = nv.new_status(torch.device("cuda")).repeat(len(self.views), 1)
        for v, (a, n_rows) in enumerate(self.slices):
            tail = (nv.ptr(off[a:]), nv.ptr(out)) if shrink is not None else ()
            nv.check(fn(nv.ptr(self.bases[v]), self.bases[v].numel(), nv.ptr(self.d_starts[a:]), nv.ptr(self.d_lens[a:]),
                        n_rows, self.enc.mode, nv.ptr(self.lut), *params, *tail, nv.ptr(status[v]), nv.stream_ptr()))
        return out, status

    def check_status(self, status, n_values=None):
        w = status.cpu().numpy()
        assert (w[:, nv.ST_BAD_BASE] == INT64_MAX).all()
        assert w[:, nv.ST_N_BASES].sum() == self.lens.sum()
        if n_values is not None:
            assert w[:, nv.ST_N_VALUES].sum() == n_values


def edge_layout(enc, span, seed):
    """16 views at byte offsets 0..15 from an aligned allocation.  View b has 9 rows on segment edges (length class c:
    edge c // 3, minus one, exactly, plus one): row 0 at the view's first byte, row c > 0 with its first byte at
    address 3b + 5c mod 16, so every address mod 16 meets every length class and the rows start at every residue
    mod 16 of their view.  Then a duplicated row, two rows overlapping it, empty rows, rows shorter than the span,
    short random rows and a last row that ends on the view's last byte (a view size that is not a multiple of 16).
    Rows come unsorted; poison between them."""
    rng = np.random.default_rng(seed)
    views, view_rows, pos = [], [], 0
    for b in range(16):
        rows, cursor = [], 0
        for c in range(9):
            s = 0 if c == 0 else cursor + 1 + (2 * b + 5 * c - cursor - 1) % 16
            rows.append((s, segment_edges((b + s) % 16, span)[c // 3] + c % 3 - 1))
            cursor = s + rows[-1][1]
        s, L = rows[int(rng.integers(9))]
        rows += [(s, L), (s + L // 3, L - L // 3), (s + 5, L - 12)]
        rows += [(int(rng.integers(0, cursor)), 0) for _ in range(2)]
        for L in list(rng.integers(1, span, size=3) if span > 1 else []) + list(rng.integers(0, 300, size=3)):
            s = cursor + 1 + int(rng.integers(0, 16))
            rows.append((s, int(L)))
            cursor = s + int(L)
        s, L = cursor + 1 + int(rng.integers(0, 16)), int(rng.integers(span, span + 100))
        L += (s + L) % 16 == 0
        rows.append((s, L))                            # the last row ends on the view's last byte
        size = s + L
        assert size % 16
        rows = [rows[i] for i in rng.permutation(len(rows))]
        vs = pos + b
        views.append((vs, size))
        view_rows.append(rows)
        pos = -(-(vs + size + 48) // 16) * 16
    return Ragged(enc, views, view_rows, rng)


@functools.lru_cache(maxsize=6)
def layout(enc_name, span):
    enc = AMINO_ENC if enc_name == "amino" else ENCODINGS[enc_name]
    return edge_layout(enc, span, seed=1000 * (ENC_NAMES + ["amino"]).index(enc_name) + span)


def prefill(bins):
    return (torch.arange(bins, dtype=torch.int64, device="cuda") * 40503) % 65521


def table_pairs(keys, counts):
    """(sorted keys, their counts, number of occupied slots) of a table, on the host."""
    keep = keys >= 0
    k, order = torch.sort(keys[keep])
    return k.cpu().numpy(), counts[keep][order].cpu().numpy(), int(keep.sum())


def new_table(cap):
    return (torch.full((cap,), -1, dtype=torch.int64, device="cuda"), torch.zeros(cap, dtype=torch.int64, device="cuda"),
            torch.zeros(1, dtype=torch.int64, device="cuda"))


# ---------------------------------------------------------------------------------------------------------------
# every entry point, every encoding, rows on segment edges
# ---------------------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("enc_name", ENC_NAMES + ["amino"])
def test_rows_encode(enc_name):
    """Codes of every row, gathered; in LUT mode the full table value (any alphabet size)."""
    lay = layout(enc_name, 1)
    out, st = lay.run(nv.lib().bnpk_rows_encode, (), shrink=0, dtype=torch.uint8)
    assert np.array_equal(out.cpu().numpy(), lay.codes)
    lay.check_status(st)


@gpu
@pytest.mark.parametrize("k", [1, 2, 15, 16, 17, 31])
@pytest.mark.parametrize("enc_name", ENC_NAMES)
def test_rows_kmer_hash(enc_name, k):
    lay = layout(enc_name, k)
    want, _ = o.get_kmers(lay.codes, lay.lens, k)
    out, st = lay.run(nv.lib().bnpk_rows_kmer_hash, (k,), shrink=k - 1)
    assert np.array_equal(out.cpu().numpy(), want)
    lay.check_status(st, want.size)


@gpu
@pytest.mark.parametrize("enc_name,cx", CANONICAL)
def test_rows_kmer_hash_canonical(enc_name, cx):
    for k in (1, 2, 15, 16, 17, 31):
        lay = layout(enc_name, k)
        want, _ = o.canonical_kmers(lay.codes, lay.lens, k, CX_ALPHABET[cx])
        out, st = lay.run(nv.lib().bnpk_rows_kmer_hash_canonical, (k, cx), shrink=k - 1)
        assert np.array_equal(out.cpu().numpy(), want), k
        lay.check_status(st, want.size)


@gpu
@pytest.mark.parametrize("k", [1, 5, 16, 31])
@pytest.mark.parametrize("enc_name", ENC_NAMES)
def test_rows_minimizers(enc_name, k):
    """Windows of 1, 2, 31, 32 k-mers (warp shuffle), 33 and 100 k-mers and 1024 bases (one lane per window)."""
    for window in [k + w - 1 for w in (1, 2, 31, 32, 33, 100)] + [1024]:
        lay = layout(enc_name, window)
        want, _ = o.get_minimizers_fast(lay.codes, lay.lens, k, window)
        out, st = lay.run(nv.lib().bnpk_rows_minimizers, (k, window), shrink=window - 1)
        assert np.array_equal(out.cpu().numpy(), want), window
        lay.check_status(st, want.size)


def count_bins(k):
    """4^k, the powers of two around it (the 32-bit fast path masks with min(bins, 4^k) - 1), shared-memory tables
    below, at and above the 32768-bin limit, and global tables."""
    bins = {30000, 32768, 32769, 77777, 1 << 22}
    if 4 ** k <= 1 << 22:
        bins |= {4 ** k, 4 ** k // 2, 4 ** k * 2}
    return sorted(bins)


@gpu
@pytest.mark.parametrize("kind", ["kmers", "minimizers", "canonical"])
@pytest.mark.parametrize("enc_name", ENC_NAMES)
def test_rows_kmer_count(enc_name, kind):
    """Every table size in every hist_mode it allows, each into a pre-filled histogram; N_VALUES and N_BASES."""
    lib = nv.lib()
    cx = CX_OF[ENCODINGS[enc_name].alphabet]
    window_of = {5: 35, 7: 46, 31: 61}                 # 31 and 40 k-mers per window: both minimizer paths
    for k in (5, 7, 31):
        window = window_of[k] if kind == "minimizers" else 0
        lay = layout(enc_name, window or k)
        if kind == "canonical":
            want, _ = o.canonical_kmers(lay.codes, lay.lens, k, CX_ALPHABET[cx])
        elif window:
            want, _ = o.get_minimizers_fast(lay.codes, lay.lens, k, window)
        else:
            want, _ = o.get_kmers(lay.codes, lay.lens, k)
        for bins in count_bins(k):
            expected = prefill(bins) + torch.from_numpy(o.count_bucketed_flat(want, bins)).cuda()
            modes = [nv.HIST_AUTO, nv.HIST_GLOBAL] + ([nv.HIST_SMEM] if bins <= nv.SMEM_MAX_BINS else [])
            for mode in modes:
                hist = prefill(bins)
                if kind == "canonical":
                    _, st = lay.run(lib.bnpk_rows_kmer_count_canonical, (k, cx, bins, mode, nv.ptr(hist)))
                else:
                    _, st = lay.run(lib.bnpk_rows_kmer_count, (k, window, bins, mode, nv.ptr(hist)))
                assert torch.equal(hist, expected), (k, bins, mode)
                lay.check_status(st, want.size)


@gpu
@pytest.mark.parametrize("enc_name,cx", [(e, 0) for e in ENC_NAMES] + CANONICAL)
def test_rows_kmer_table_insert_and_rehash(enc_name, cx):
    """Keys and counts equal np.unique; a second insert doubles the counts; growth into 2x and 8x keeps them."""
    lib = nv.lib()
    k = 21
    lay = layout(enc_name, k)
    want = o.canonical_kmers(lay.codes, lay.lens, k, CX_ALPHABET[cx])[0] if cx else o.get_kmers(lay.codes, lay.lens, k)[0]
    u, c = np.unique(want, return_counts=True)
    cap = 1 << 22
    assert 2 * want.size <= cap
    keys, counts, used = new_table(cap)
    for times in (1, 2):
        _, st = lay.run(lib.bnpk_rows_kmer_table_insert, (k, cx, nv.ptr(keys), nv.ptr(counts), cap, nv.ptr(used)))
        lay.check_status(st, want.size)
        assert not st[:, nv.ST_TABLE_FULL].any()
        gk, gc, n = table_pairs(keys, counts)
        assert np.array_equal(gk, u) and np.array_equal(gc, times * c) and n == int(used.item()) == u.size
    for grow in (2, 8):
        nk, nc, nu = new_table(cap * grow)
        status = nv.new_status(torch.device("cuda"))
        nv.check(lib.bnpk_kmer_table_rehash(nv.ptr(keys), nv.ptr(counts), cap, nv.ptr(nk), nv.ptr(nc), cap * grow,
                                            nv.ptr(nu), nv.ptr(status), nv.stream_ptr()))
        gk, gc, n = table_pairs(nk, nc)
        assert np.array_equal(gk, u) and np.array_equal(gc, 2 * c) and n == int(nu.item()) == u.size
        assert int(status[nv.ST_TABLE_FULL].item()) == 0


def _kmer_rows(keys_and_times, k):
    """ACGT text rows of exactly k bases, one per occurrence of a k-mer hash, laid out with poison between them."""
    strings = [o.kmer_to_string(int(h), k) for h, t in keys_and_times for _ in range(int(t))]
    starts = np.arange(len(strings), dtype=np.int64) * (k + 3)
    host = np.full(len(strings) * (k + 3), ord("N"), dtype=np.uint8)
    for s, text in zip(starts, strings):
        host[s: s + k] = np.frombuffer(text.encode(), dtype=np.uint8)
    lens = np.full(len(strings), k, dtype=np.int32)
    return host, starts, lens


def _insert(host, starts, lens, k, cap):
    from bionumpy_b200 import ops
    keys, counts, used = new_table(cap)
    st = ops.rows_kmer_table_insert(torch.from_numpy(host).cuda(), torch.from_numpy(starts).cuda(),
                                    torch.from_numpy(lens).cuda(), nv.ENC_ASCII_ACGT, k, keys, counts, used)
    return keys.cpu().numpy(), counts.cpu().numpy(), int(used.item()), st.cpu().numpy()


@gpu
def test_small_table_probe_wraps_past_the_last_slot():
    """Four k-mers whose home is the last of 64 slots: all but one probe on from slot 0.  Every key sits after a run
    of occupied slots that starts at its home."""
    k, cap = 7, 64
    rng = np.random.default_rng(64)
    all_h = np.arange(4 ** k, dtype=np.uint64)
    home = (o.splitmix64(all_h) & np.uint64(cap - 1)).astype(np.int64)
    chosen = np.concatenate([all_h[home == cap - 1][:4], rng.choice(all_h[home != cap - 1], 26, replace=False)])
    times = rng.integers(1, 5, size=chosen.size)
    host, starts, lens = _kmer_rows(zip(chosen, times), k)
    keys, counts, used, st = _insert(host, starts, lens, k, cap)
    want = o.get_kmers(o.encode_flat(o.gather_rows(host, starts, lens), o.alphabet_lut()), lens, k)[0]
    u, c = np.unique(want, return_counts=True)
    occ = keys >= 0
    order = np.argsort(keys[occ])
    assert np.array_equal(keys[occ][order], u) and np.array_equal(counts[occ][order], c) and used == u.size == 30
    assert st[nv.ST_TABLE_FULL] == 0 and st[nv.ST_BAD_BASE] == INT64_MAX
    wrapped = 0
    for slot in np.flatnonzero(occ):
        h = int(o.splitmix64(np.array([keys[slot]], dtype=np.uint64))[0]) & (cap - 1)
        assert all(occ[(h + j) % cap] for j in range((slot - h) % cap))
        wrapped += slot < h
    assert wrapped >= 3


@gpu
def test_full_table_keeps_exact_counts_of_the_keys_it_holds():
    """40 distinct k-mers into 16 slots: word 13 is set, every slot is used, and every key present has its count."""
    k, cap = 7, 16
    rng = np.random.default_rng(16)
    chosen = rng.choice(4 ** k, 40, replace=False)
    host, starts, lens = _kmer_rows(zip(chosen, rng.integers(1, 6, size=40)), k)
    keys, counts, used, st = _insert(host, starts, lens, k, cap)
    want = o.get_kmers(o.encode_flat(o.gather_rows(host, starts, lens), o.alphabet_lut()), lens, k)[0]
    u, c = np.unique(want, return_counts=True)
    assert st[nv.ST_TABLE_FULL] != 0 and used == cap and (keys >= 0).all()
    assert len(set(keys.tolist())) == cap
    idx = np.searchsorted(u, keys)
    assert np.array_equal(u[idx], keys) and np.array_equal(c[idx], counts)


# ---------------------------------------------------------------------------------------------------------------
# the generic-alphabet hash (int64 wrap-around), reverse complement, bincounts
# ---------------------------------------------------------------------------------------------------------------
def _scattered_rows(rng, lens, poison, letters, view_off):
    """Rows at every residue mod 16 with poison between them, in a view view_off bytes into an aligned buffer."""
    starts, cursor = [], 0
    for i, L in enumerate(lens):
        cursor += 1 + (i * 7 - cursor - 1 - view_off) % 16
        starts.append(cursor)
        cursor += int(L)
    host = np.full(view_off + cursor + 16, poison, dtype=np.uint8)
    for s, L in zip(starts, lens):
        host[view_off + s: view_off + s + L] = rng.choice(letters, size=int(L))
    return host, np.array(starts, dtype=np.int64), np.asarray(lens, dtype=np.int32)


def generic_hashes(code_rows, k, a):
    """sum_j code[i+j] * a^j modulo 2^64 in Python integers, as int64."""
    powers = [pow(a, j, 1 << 64) for j in range(k)]
    out = []
    for c in code_rows:
        for i in range(len(c) - k + 1):
            h = sum(x * p for x, p in zip(c[i:i + k], powers)) & ((1 << 64) - 1)
            out.append(h - (1 << 64) if h >> 63 else h)
    return np.array(out, dtype=np.int64)


@gpu
@pytest.mark.parametrize("alphabet_size", [2, 3, 5, 20, 21, 255])
def test_rows_generic_hash(alphabet_size):
    """k up to 63 on rows longer than a warp, with and without a LUT; the first invalid symbol as (row, position)."""
    from bionumpy_b200 import ops
    a = alphabet_size
    rng = np.random.default_rng(a)
    lens = [0, 1, 31, 32, 33, 62, 63, 64, 65, 100, 130, 200] + [int(x) for x in rng.integers(0, 150, size=6)]
    for use_lut in (False, True):
        if use_lut:
            perm = rng.permutation(256).astype(np.uint8)
            lut = np.full(256, 255, dtype=np.uint8)
            lut[perm[:a]] = np.arange(a)
            letters, poison = perm[:a], perm[a]
        else:
            lut, letters, poison = None, np.arange(a, dtype=np.uint8), min(a, 255)
        host, starts, lens_a = _scattered_rows(rng, lens, poison, letters, view_off=5)
        rows = [host[5 + s: 5 + s + L] for s, L in zip(starts, lens_a)]
        code_rows = [[int(x) for x in (lut[r] if use_lut else r)] for r in rows]
        dev = torch.from_numpy(host).cuda()
        base, d_starts, d_lens = dev[5:], torch.from_numpy(starts).cuda(), torch.from_numpy(lens_a).cuda()
        d_lut = None if lut is None else torch.from_numpy(lut).cuda()
        for k in (1, 13, 31, 40, 63):
            out, offsets, st = ops.rows_generic_hash(base, d_starts, d_lens, a, k, d_lut)
            assert np.array_equal(out.cpu().numpy(), generic_hashes(code_rows, k, a)), (use_lut, k)
            assert ops.read_status(st).bad_base() is None
        for r, p in ((11, 3), (9, 40), (10, 99)):       # invalid symbols in three rows: the first row's is reported
            host[5 + starts[r] + p] = poison
        _, _, st = ops.rows_generic_hash(torch.from_numpy(host).cuda()[5:], d_starts, d_lens, a, 13, d_lut)
        assert ops.read_status(st).bad_base() == (9, 40)


@gpu
@pytest.mark.parametrize("alphabet", [None, "ACGT", "ACTG", "ATCG"])
def test_rows_reverse_complement(alphabet):
    """Every complement table (BaseEncoding text and the code tables), unaligned rows of up to 5000 bytes."""
    from bionumpy_b200 import ops
    rng = np.random.default_rng([None, "ACGT", "ACTG", "ATCG"].index(alphabet))
    lens = [0, 1, 15, 16, 17, 31, 32, 33, 1000, 4999, 5000] + [int(x) for x in rng.integers(0, 5001, size=20)]
    letters = np.arange(256, dtype=np.uint8) if alphabet is None else np.arange(4, dtype=np.uint8)
    host, starts, lens_a = _scattered_rows(rng, lens, 0, letters, view_off=3)
    order = rng.permutation(len(lens))                 # unsorted rows
    starts, lens_a = starts[order], lens_a[order]
    dev = torch.from_numpy(host).cuda()
    lut = torch.from_numpy(o.complement_table(alphabet)).cuda()
    out, _ = ops.rows_reverse_complement(dev[3:], torch.from_numpy(starts).cuda(), torch.from_numpy(lens_a).cuda(), lut)
    want = o.reverse_complement_rows(o.gather_rows(host[3:], starts, lens_a), lens_a, alphabet)
    assert np.array_equal(out.cpu().numpy(), want)


@gpu
@pytest.mark.parametrize("bins", [1, 64, 1000, 30000, 32768, 32769, 77777, 1 << 22])
def test_bincount_and_bincount_rows(bins):
    from bionumpy_b200 import ops
    rng = np.random.default_rng(bins)
    values = rng.integers(0, 1 << 62, size=300_000)
    d_values = torch.from_numpy(values).cuda()
    want = prefill(bins) + torch.from_numpy(o.count_bucketed_flat(values, bins)).cuda()
    for mode in [nv.HIST_AUTO, nv.HIST_GLOBAL] + ([nv.HIST_SMEM] if bins <= nv.SMEM_MAX_BINS else []):
        hist, st = ops.bincount(d_values, bins, hist=prefill(bins), hist_mode=mode)
        assert torch.equal(hist, want), mode
        assert int(st[nv.ST_BAD_BASE].item()) == INT64_MAX
        neg = values.copy()
        neg[[200_001, 77_777, 150_000]] = [-1, -(1 << 62), -5]
        _, st = ops.bincount(torch.from_numpy(neg).cuda(), bins, hist_mode=mode)
        assert int(st[nv.ST_BAD_BASE].item()) == 77_777
    if bins <= 77777:
        lens = rng.integers(0, 60, size=40).astype(np.int32)
        vals = rng.integers(0, 1 << 62, size=int(lens.sum()))
        offsets = ops.row_offsets(torch.from_numpy(lens).cuda())
        out, st = ops.bincount_rows(torch.from_numpy(vals).cuda(), offsets, bins)
        assert np.array_equal(out.cpu().numpy(), o.count_rows(vals % bins, lens, bins))
        assert int(st[nv.ST_BAD_BASE].item()) == INT64_MAX
        vals[[vals.size // 2, vals.size // 3]] = -3
        _, st = ops.bincount_rows(torch.from_numpy(vals).cuda(), offsets, bins)
        assert int(st[nv.ST_BAD_BASE].item()) == vals.size // 3


# ---------------------------------------------------------------------------------------------------------------
# bad bytes across segments, every mode and encoding
# ---------------------------------------------------------------------------------------------------------------
BAD_MODES = {  # name: (k, window)
    "encode": (1, 0), "hash": (21, 0), "canonical": (21, 0), "minimizers": (15, 40), "minimizers_long": (5, 100),
    "count": (21, 0), "count_canonical": (21, 0), "count_minimizers": (15, 40), "table": (21, 0),
}
PLACEMENTS = ["overlap", "after_overlap", "after_second_overlap", "last_byte_first_edge", "last_byte_second_edge",
              "two_rows"]
TARGET = 2


def bad_case(enc, span, placement, i, rng):
    """One view: rows 60, 0, the target row, 40 and 2100 bytes long; the target row starts at a varying address mod 16
    and holds the bad byte (two_rows: the target row late in a segment, row 4 early in its first)."""
    view_off, a = i % 16, (5 * i + 3) % 16
    e = segment_edges(a, span)
    length, bad = e[2] + 10, []
    if placement == "overlap":
        bad = [(TARGET, e[0] - (span - 1) + (span - 1) // 2)]
    elif placement == "after_overlap":
        bad = [(TARGET, e[0])]
    elif placement == "after_second_overlap":
        bad = [(TARGET, e[1])]
    elif placement == "last_byte_first_edge":
        length, bad = e[0], [(TARGET, e[0] - 1)]
    elif placement == "last_byte_second_edge":
        length, bad = e[1], [(TARGET, e[1] - 1)]
    else:
        bad = [(4, 3), (TARGET, e[0] + 7)]
    rows, cursor = [], 0
    for r, L in enumerate([60, 0, length, 40, 2100]):
        s = cursor + 1 + ((a - view_off - cursor - 1) % 16 if r == TARGET else int(rng.integers(0, 16)))
        rows.append((s, L))
        cursor = s + L
    return Ragged(enc, [(view_off, cursor)], [rows], rng, bad=[(0, r, p) for r, p in bad])


def run_mode(lay, mode, k, window, cx):
    lib = nv.lib()
    if mode == "encode":
        return lay.run(lib.bnpk_rows_encode, (), shrink=0, dtype=torch.uint8)[1]
    if mode == "hash":
        return lay.run(lib.bnpk_rows_kmer_hash, (k,), shrink=k - 1)[1]
    if mode == "canonical":
        return lay.run(lib.bnpk_rows_kmer_hash_canonical, (k, cx), shrink=k - 1)[1]
    if mode.startswith("minimizers"):
        return lay.run(lib.bnpk_rows_minimizers, (k, window), shrink=window - 1)[1]
    hist = torch.zeros(4096, dtype=torch.int64, device="cuda")
    if mode == "count_canonical":
        return lay.run(lib.bnpk_rows_kmer_count_canonical, (k, cx, 4096, nv.HIST_AUTO, nv.ptr(hist)))[1]
    if mode.startswith("count"):
        return lay.run(lib.bnpk_rows_kmer_count, (k, window, 4096, nv.HIST_AUTO, nv.ptr(hist)))[1]
    keys, counts, used = new_table(1 << 15)
    return lay.run(lib.bnpk_rows_kmer_table_insert, (k, cx, nv.ptr(keys), nv.ptr(counts), 1 << 15, nv.ptr(used)))[1]


def oracle_bad_base(lay):
    """The oracle's first invalid byte of the gathered rows as (row, position in row)."""
    try:
        o.encode_flat(lay.flat, lay.enc.table, lay.enc.size)
    except o.OracleEncodingError as e:
        ends = np.cumsum(lay.lens.astype(np.int64))
        row = int(np.searchsorted(ends, e.offset, side="right"))
        return row, int(e.offset - (ends[row] - lay.lens[row]))
    return None


@gpu
@pytest.mark.parametrize("enc_name", ENC_NAMES)
def test_bad_bytes_across_segments(enc_name):
    """A bad byte in a segment overlap, on the first byte after one, on the last byte of a row that ends on a segment
    edge, and in two rows at once: every mode reports the oracle's minimum (row << 32 | position)."""
    enc = ENCODINGS[enc_name]
    cx = CX_OF[enc.alphabet]
    rng = np.random.default_rng(77 + ENC_NAMES.index(enc_name))
    cases, i = [], 0
    for mode, (k, window) in BAD_MODES.items():
        for placement in PLACEMENTS:
            span = window or k
            if placement == "overlap" and span == 1:
                continue
            lay = bad_case(enc, span, placement, i, rng)
            i += 1
            want = oracle_bad_base(lay)
            assert want is not None and want[0] == TARGET
            cases.append(((mode, placement), run_mode(lay, mode, k, window, cx), want))
    words = torch.stack([st[0] for _, st, _ in cases]).cpu().numpy()
    for (label, _, want), w in zip(cases, words):
        assert w[nv.ST_BAD_BASE] == (want[0] << 32 | want[1]), label


# ---------------------------------------------------------------------------------------------------------------
# the Python layer's long-row split
# ---------------------------------------------------------------------------------------------------------------
def split_lengths(piece, span):
    return [piece + span - 2, piece + span - 1, piece + span, 2 * piece + span - 1, 0, min(span, 3), 2 * piece + span]


@pytest.mark.parametrize("piece,span", [(16384, 1), (16384, 21), (16384, 1024), (7, 1), (7, 2), (7, 5), (7, 8)])
def test_split_long_rows_puts_every_window_start_in_one_piece(piece, span):
    from bionumpy_b200.sequence.kmers import _split_long_rows
    lens = np.array(split_lengths(piece, span), dtype=np.int64)
    starts = np.cumsum(lens + 3) - lens - 3 + 1
    n_win = np.maximum(lens - span + 1, 0)
    offsets = np.concatenate([[0], np.cumsum(n_win)])
    ps, pl, po = _split_long_rows(torch.from_numpy(starts), torch.from_numpy(lens.astype(np.int32)), span,
                                  torch.from_numpy(offsets), piece=piece)
    ps, pl, po = ps.numpy(), pl.numpy().astype(np.int64), po.numpy()
    assert ps.size == pl.size == po.size
    windows = np.zeros(int(offsets[-1]), dtype=np.int64)
    bytes_seen = [np.zeros(L, dtype=bool) for L in lens]
    for s, L, off in zip(ps, pl, po):
        r = int(np.searchsorted(starts, s, side="right")) - 1
        rel = s - starts[r]
        assert 0 <= rel and rel + L <= lens[r] and L <= piece + span - 1
        assert off == offsets[r] + rel                 # the piece's first window is the row's window rel
        windows[off: off + max(L - span + 1, 0)] += 1
        bytes_seen[r][rel: rel + L] = True
    assert (windows == 1).all()
    assert all(b.all() for b in bytes_seen)            # every byte is read, so a bad one is still found
    short = torch.from_numpy(lens[:2].astype(np.int32))
    same = _split_long_rows(torch.from_numpy(starts[:2]), short, span, None, piece=piece)
    assert same[1] is short


@gpu
@pytest.mark.parametrize("k,window", [(21, 0), (31, 0), (15, 40)])
def test_api_on_rows_cut_into_pieces(k, window):
    """get_kmers (plain and canonical) / get_minimizers, count_kmers_hashed and count_kmers_exact on rows around the
    piece length; a bad byte that only the second piece of a row holds raises EncodingError with the oracle's offset."""
    import bionumpy_b200 as bnp
    from bionumpy_b200.sequence.kmers import LONG_ROW
    span = window or k
    lens = split_lengths(LONG_ROW, span)
    rng = np.random.default_rng(span)
    strings = ["".join(rng.choice(list("ACGTacgt"), size=L)) for L in lens]
    flat = np.frombuffer("".join(strings).encode(), dtype=np.uint8)
    codes = o.encode_flat(flat, o.alphabet_lut())
    L = np.array(lens, dtype=np.int64)

    def as_codes(c):
        return bnp.EncodedRaggedArray(bnp.EncodedArray(torch.from_numpy(c.copy()).cuda(), bnp.DNAEncoding), lens)

    text = bnp.as_encoded_array(strings)
    if window:
        want, wl = o.get_minimizers_fast(codes, L, k, window)
        got = bnp.get_minimizers(as_codes(codes), k, window)
    else:
        want, wl = o.get_kmers(codes, L, k)
        got = bnp.get_kmers(text, k)
    assert np.array_equal(got.raw().ravel().cpu().numpy(), want) and got.lengths.cpu().tolist() == wl.tolist()
    B = 1 << 16
    assert np.array_equal(bnp.count_kmers_hashed(text, k, B, window_size=window).cpu().numpy(),
                          o.count_bucketed_flat(want, B))
    if not window:
        want_c, _ = o.canonical_kmers(codes, L, k)
        assert np.array_equal(bnp.get_kmers(text, k, canonical=True).raw().ravel().cpu().numpy(), want_c)
        u, c = np.unique(want, return_counts=True)
        got_t = bnp.count_kmers_exact(text, k)
        assert np.array_equal(got_t.kmers.cpu().numpy(), u) and np.array_equal(got_t.counts.cpu().numpy(), c)

    pos = LONG_ROW + span + 3                          # past the first piece of row 3
    assert pos >= LONG_ROW + span - 1
    bad_strings = list(strings)
    bad_strings[3] = strings[3][:pos] + "N" + strings[3][pos + 1:]
    with pytest.raises(o.OracleEncodingError) as want_err:
        o.encode_flat(np.frombuffer("".join(bad_strings).encode(), dtype=np.uint8), o.alphabet_lut())
    bad_text = bnp.as_encoded_array(bad_strings)
    bad_codes = codes.copy()
    bad_codes[want_err.value.offset] = 7
    calls = [lambda: bnp.count_kmers_hashed(bad_text, k, B, window_size=window)]
    if window:
        calls.append(lambda: bnp.get_minimizers(as_codes(bad_codes), k, window).raw())
    else:
        calls += [lambda: bnp.get_kmers(bad_text, k).raw(), lambda: bnp.get_kmers(bad_text, k, canonical=True).raw(),
                  lambda: bnp.count_kmers_exact(bad_text, k),
                  lambda: bnp.count_kmers_hashed(as_codes(bad_codes), k, B)]
    for call in calls:
        with pytest.raises(bnp.EncodingError) as got_err:
            call()
        assert got_err.value.offset == want_err.value.offset


# ---------------------------------------------------------------------------------------------------------------
# argument checks (CPU): each entry point returns its BNPK_E_* code before any CUDA call.  n_rows = 0 makes a
# valid call return 0 without touching the device, so the pointers are never read.
# ---------------------------------------------------------------------------------------------------------------
def test_row_entry_points_reject_bad_arguments():
    lib = nv.load_library()
    N = None
    LUT = 16                                           # any non-null pointer: with no rows it is never read
    A, CODES = nv.ENC_ASCII_ACGT, nv.ENC_CODES
    BAD, EK, EW, EB = nv.E_BADARG, nv.E_K, nv.E_WINDOW, nv.E_BINS
    rows = (N, 0, N, N, 0)

    def enc(mode, lut=N):
        return lib.bnpk_rows_encode(*rows, mode, lut, N, N, N, N)

    def khash(k, mode=A, lut=N):
        return lib.bnpk_rows_kmer_hash(*rows, mode, lut, k, N, N, N, N)

    def ghash(a, k, lut=N):
        return lib.bnpk_rows_generic_hash(*rows, lut, a, k, N, N, N, N)

    def mins(k, w, mode=A, lut=N):
        return lib.bnpk_rows_minimizers(*rows, mode, lut, k, w, N, N, N, N)

    def count(k, w=0, bins=64, hm=nv.HIST_AUTO, mode=A, lut=N):
        return lib.bnpk_rows_kmer_count(*rows, mode, lut, k, w, bins, hm, N, N, N)

    def chash(k, cx, mode=A, lut=N):
        return lib.bnpk_rows_kmer_hash_canonical(*rows, mode, lut, k, cx, N, N, N, N)

    def ccount(k, cx, bins=64, hm=nv.HIST_AUTO, mode=A, lut=N):
        return lib.bnpk_rows_kmer_count_canonical(*rows, mode, lut, k, cx, bins, hm, N, N, N)

    def table(k, cx, cap=64, mode=A, lut=N):
        return lib.bnpk_rows_kmer_table_insert(*rows, mode, lut, k, cx, N, N, cap, N, N, N)

    for mode in (-1, 4):
        assert enc(mode) == khash(21, mode) == mins(5, 9, mode) == count(5, 0, 64, 0, mode) == BAD
        assert chash(5, 3, mode) == ccount(5, 3, 64, 0, mode) == table(5, 0, 64, mode) == BAD
    assert enc(nv.ENC_LUT) == khash(21, nv.ENC_LUT) == mins(5, 9, nv.ENC_LUT) == count(5, mode=nv.ENC_LUT) == BAD
    assert chash(5, 3, nv.ENC_LUT) == ccount(5, 3, mode=nv.ENC_LUT) == table(5, 0, mode=nv.ENC_LUT) == BAD
    assert enc(nv.ENC_LUT, LUT) == khash(21, nv.ENC_LUT, LUT) == count(5, mode=nv.ENC_LUT, lut=LUT) == 0
    assert enc(CODES) == 0
    for k in (0, 32):
        assert khash(k) == mins(k, 40) == count(k) == count(k, 40) == chash(k, 3) == ccount(k, 3) == table(k, 0) == EK
    for k in (1, 31):
        assert khash(k) == mins(k, 31) == count(k) == chash(k, 3) == ccount(k, 3) == table(k, 3) == 0
    assert mins(5, 4) == count(5, 4) == mins(5, 1025) == count(5, 1025) == mins(5, 0) == EW
    assert mins(5, 1024) == count(5, 1024) == mins(5, 5) == 0
    for cx in (0, 4):
        assert chash(5, cx) == ccount(5, cx) == BAD
    assert table(5, -1) == table(5, 4) == table(5, 0, cap=48) == BAD
    assert all(chash(5, cx) == ccount(5, cx) == table(5, cx) == 0 for cx in (1, 2, 3))
    assert count(5, 0, 32769, nv.HIST_SMEM) == count(5, 9, 32769, nv.HIST_SMEM) == ccount(5, 3, 32769, nv.HIST_SMEM) == EB
    assert count(5, 0, 0) == ccount(5, 3, 0) == EB
    assert count(5, 0, 32768, nv.HIST_SMEM) == ccount(5, 3, 32768, nv.HIST_SMEM) == count(5, 0, 32769) == 0
    assert ghash(21, 0) == ghash(21, 64) == EK
    assert ghash(1, 5) == ghash(256, 5) == BAD
    assert ghash(2, 63) == ghash(255, 1) == ghash(21, 5, LUT) == 0
    assert lib.bnpk_rows_reverse_complement(*rows, N, N, N, N) == BAD
    assert lib.bnpk_rows_reverse_complement(*rows, LUT, N, N, N) == 0
    assert lib.bnpk_bincount(N, 0, 32769, nv.HIST_SMEM, N, N, N) == lib.bnpk_bincount(N, 0, 0, 0, N, N, N) == EB
    assert lib.bnpk_bincount(N, 0, 32768, nv.HIST_SMEM, N, N, N) == 0
    assert lib.bnpk_bincount_rows(N, N, 0, 0, N, N, N) == EB


def test_row_kernels_have_no_stack_frame():
    """Every build of the row kernel the row entry points launch, and the other row and bincount kernels, is sm_90a
    code without local memory."""
    from bionumpy_b200 import _native
    tool = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(tool):
        pytest.skip("cuobjdump not available")
    out = subprocess.run([tool, "-res-usage", _native.LIB_PATH], capture_output=True, text=True).stdout
    assert "sm_90a" in out
    usage = dict(re.findall(r"Function (\S+):\s*REG:\d+ STACK:(\d+)", out))
    rows = [n for n in usage if re.match(r"_ZN4bnpk11rows_kernelILi\dELi\dELb[01]ELb0EEEvNS_7RowArgsE$", n)]
    assert len(rows) == 32                             # 6 modes x 4 encodings, and both table kinds of the 2 counts
    others = [n for n in usage if re.match(r"_ZN4bnpk(14uncount_kernel|24rows_generic_hash_kernel|"
                                           r"30rows_reverse_complement_kernel|19table_rehash_kernel|15bincount_kernel)", n)]
    assert len(others) == 8 + 1 + 1 + 1 + 2
    for name in rows + others:
        assert usage[name] == "0", name
