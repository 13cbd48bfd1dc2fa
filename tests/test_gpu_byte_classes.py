"""Every byte value through every kernel that classifies sequence bytes, in every encoding.

Each route must report the oracle's BAD_BASE (entry and offset) for a byte outside the alphabet, and for a valid byte
no error and the oracle's histogram.  One case is one byte value in one sequence line of a small FASTQ chunk.  Across
byte values the byte goes to the row's first unit, an interior unit and its last unit, and the row start varies so
that the byte lands on all 16 positions of a 16-byte unit.  The interior unit lies in the steady state of the
warp-specialised count (whole units), the other two in its masked encode.  Every case has its own status block, and
all of them are read once at the end."""
from collections import namedtuple

import numpy as np
import pytest
import torch

from oracle import bnp_oracle as o
from test_gpu_sliced_count import ROUTES

gpu = pytest.mark.gpu

ENC_ACGT, ENC_ACTG, ENC_CODES, ENC_LUT = 0, 1, 2, 3
N_RECORDS, TARGET, ROW_LEN = 40, 3, 150          # rows 0..31 share one 32-row chunk of the warp-specialised count
LONG_ROW = 1500                                  # longer than the 1024-byte row walk: counted by the deferred pass
Encoding = namedtuple("Encoding", "mode lut alphabet")      # alphabet: the oracle's table (codes, validity)


def _codes_lut():
    lut = np.full(256, 255, dtype=np.uint8)
    lut[:4] = np.arange(4)
    return lut


ENCODINGS = {
    "acgt": Encoding(ENC_ACGT, None, o.alphabet_lut("ACGT")),
    "actg": Encoding(ENC_ACTG, None, o.alphabet_lut("ACTG")),
    "codes": Encoding(ENC_CODES, None, _codes_lut()),
    "lut_acgt": Encoding(ENC_LUT, o.alphabet_lut("ACGT"), o.alphabet_lut("ACGT")),
    "lut_actg": Encoding(ENC_LUT, o.alphabet_lut("ACTG"), o.alphabet_lut("ACTG")),
}
BYTES = [v for v in range(256) if v != 10]


def placement(v, row_len):
    """(row start mod 16, row length, offset of the byte in the row) for byte value v: the byte sits at position
    v % 16 of the row's first unit, its fifth unit or its last unit."""
    ph, place = v % 16, (v // 16) % 3
    if place == 0:
        r = (v // 48) % (ph + 1)
        return r, row_len, ph - r
    if place == 1:
        r = (5 * v) % 16
        return r, row_len, 64 + ph - r
    r = (v // 48) % 16
    length = row_len + (15 - (r + row_len - 1)) % 16        # the row ends at position 15 of its last unit
    return r, length, length - 16 + ph


def build_chunk(enc_name, v, row_len=ROW_LEN):
    """A FASTQ chunk whose record TARGET holds byte v; returns (chunk, offset of v in that row)."""
    rng = np.random.default_rng(1000 + v)
    alphabet = np.arange(4, dtype=np.uint8) if enc_name == "codes" else np.frombuffer(b"ACGTacgt", dtype=np.uint8)
    r, length, pos = placement(v, row_len)
    parts, size = [], 0
    for i in range(N_RECORDS):
        L = length if i == TARGET else ROW_LEN
        seq = rng.choice(alphabet, size=L)
        header = b"@r%d" % i
        if i == TARGET:
            header += b"x" * ((r - (size + len(header) + 1)) % 16)
            seq[pos] = v
        qual = rng.integers(33, 74, size=L, dtype=np.uint8).tobytes()
        rec = header + b"\n" + seq.tobytes() + b"\n+\n" + qual + b"\n"
        parts.append(rec)
        size += len(rec)
    chunk = np.frombuffer(b"".join(parts), dtype=np.uint8).copy()
    _, starts, _ = o.fastq_split(chunk)
    assert starts[TARGET, 1] % 16 == r and chunk[starts[TARGET, 1] + pos] == v
    return chunk, pos


def oracle_values(chunk, enc, k, window):
    """The k-mer or minimizer values of the chunk's sequence lines under the encoding (all bytes valid)."""
    _, starts, lens = o.fastq_split(chunk)
    codes = o.encode_flat(o.gather_rows(chunk, starts[:, 1], lens[:, 1]), enc.alphabet)
    return (o.get_minimizers_fast(codes, lens[:, 1], k, window) if window else o.get_kmers(codes, lens[:, 1], k))[0]


class Cases:
    """Launches on one stream, one status block per case, and histogram checks that stay on the device."""

    def __init__(self):
        from bionumpy_b200 import _native as nv
        self.nv = nv
        self.status0 = nv.new_status(torch.device("cuda"))
        self.status, self.mismatch, self.want = [], [], []

    def new_status(self, label, want_bad):
        st = self.status0.clone()
        self.status.append(st)
        self.want.append((label, want_bad))
        return st

    def check_hist(self, hist, values, bins):
        """hist must equal the oracle's count of `values` (value % bins): subtract it on the device, keep any()."""
        idx, cnt = np.unique(np.asarray(values) % bins, return_counts=True)
        hist.index_put_((torch.from_numpy(idx).cuda(),), -torch.from_numpy(cnt.astype(np.int64)).cuda(), accumulate=True)
        self.mismatch.append((len(self.status) - 1, hist.any()))

    def verify(self):
        from bionumpy_b200 import ops
        words = torch.stack(self.status).cpu()
        got = [ops.ScanStatus(w.tolist()) for w in words]
        for (label, want), s in zip(self.want, got):
            assert s.bad_base() == want, label
            assert not s.overflow, label
        for i, m in self.mismatch:
            assert not bool(m), self.want[i][0]


def upload(arrays, dtype):
    """One host-to-device copy for many small arrays: device views, each starting at a multiple of 256 bytes."""
    item = np.dtype(dtype).itemsize
    offs = np.cumsum([0] + [-(-a.nbytes // 256) * 256 // item for a in arrays])
    host = np.zeros(offs[-1], dtype=dtype)
    for a, b in zip(arrays, offs):
        host[b: b + a.size] = a
    dev = torch.from_numpy(host).cuda()
    return [dev[b: b + a.size] for a, b in zip(arrays, offs)]


def fused_count(cases, enc, lut, chunk_dev, route, label, want_bad, values):
    nv = cases.nv
    n = chunk_dev.numel()
    buf = torch.zeros(n + route.shift + 64, dtype=torch.uint8, device="cuda")
    chunk = buf[route.shift: route.shift + n]
    chunk.copy_(chunk_dev)
    hist = torch.zeros(route.bins, dtype=torch.int64, device="cuda")
    st = cases.new_status(label, want_bad)
    ws = nv.workspace(n, chunk.device)
    nv.check(nv.lib().bnpk_chunk_kmer_count(
        nv.ptr(chunk), n, 0, n, 1, 4, ord("@"), 1, -1, enc.mode, nv.ptr(lut), route.k, route.window, route.bins,
        route.hist_mode, nv.ptr(hist), nv.ptr(st), nv.ptr(ws), ws.numel(), nv.stream_ptr()))
    if want_bad is None:
        cases.check_hist(hist, values(route.k, route.window), route.bins)


K, WINDOW = 21, 31                     # the row entry points' k-mer size and minimizer window


def out_offsets(lens, span):
    """Output offsets of rows yielding L - span + 1 values each, and the total."""
    m = np.maximum(lens.astype(np.int64) - span + 1, 0)
    return np.cumsum(m) - m, int(m.sum())


def row_entry_points(cases, enc, lut, chunk_dev, starts, lens, offs, label, want_bad, values):
    """offs: {span: (device output offsets, total)} for spans 1, K and WINDOW."""
    nv = cases.nv
    lib, s = nv.lib(), nv.stream_ptr()
    n_rows = starts.numel()
    base, n = nv.ptr(chunk_dev), chunk_dev.numel()
    k, window, bins = K, WINDOW, 1 << 14

    if enc.mode != ENC_LUT:
        off, total = offs[1]
        out = torch.empty(total, dtype=torch.uint8, device="cuda")
        nv.check(lib.bnpk_rows_encode(base, n, nv.ptr(starts), nv.ptr(lens), n_rows, enc.mode, nv.ptr(lut), nv.ptr(off),
                                      nv.ptr(out), nv.ptr(cases.new_status(label + ("rows_encode",), want_bad)), s))
    off, total = offs[k]
    out = torch.empty(total, dtype=torch.int64, device="cuda")
    nv.check(lib.bnpk_rows_kmer_hash(base, n, nv.ptr(starts), nv.ptr(lens), n_rows, enc.mode, nv.ptr(lut), k, nv.ptr(off),
                                     nv.ptr(out), nv.ptr(cases.new_status(label + ("rows_kmer_hash",), want_bad)), s))
    nv.check(lib.bnpk_rows_kmer_hash_canonical(
        base, n, nv.ptr(starts), nv.ptr(lens), n_rows, enc.mode, nv.ptr(lut), k, 3, nv.ptr(off), nv.ptr(out),
        nv.ptr(cases.new_status(label + ("rows_kmer_hash_canonical",), want_bad)), s))
    off, total = offs[window]
    out = torch.empty(total, dtype=torch.int64, device="cuda")
    nv.check(lib.bnpk_rows_minimizers(base, n, nv.ptr(starts), nv.ptr(lens), n_rows, enc.mode, nv.ptr(lut), k, window,
                                      nv.ptr(off), nv.ptr(out),
                                      nv.ptr(cases.new_status(label + ("rows_minimizers",), want_bad)), s))
    hist = torch.zeros(bins, dtype=torch.int64, device="cuda")
    nv.check(lib.bnpk_rows_kmer_count(base, n, nv.ptr(starts), nv.ptr(lens), n_rows, enc.mode, nv.ptr(lut), k, 0, bins,
                                      0, nv.ptr(hist), nv.ptr(cases.new_status(label + ("rows_kmer_count",), want_bad)), s))
    if want_bad is None:
        cases.check_hist(hist, values(k, 0), bins)
    cap = 1 << 15
    keys = torch.full((cap,), -1, dtype=torch.int64, device="cuda")
    counts = torch.zeros(cap, dtype=torch.int64, device="cuda")
    used = torch.zeros(1, dtype=torch.int64, device="cuda")
    nv.check(lib.bnpk_rows_kmer_table_insert(
        base, n, nv.ptr(starts), nv.ptr(lens), n_rows, enc.mode, nv.ptr(lut), k, 0, nv.ptr(keys), nv.ptr(counts), cap,
        nv.ptr(used), nv.ptr(cases.new_status(label + ("rows_kmer_table_insert",), want_bad)), s))


def run_cases(enc_name, row_len, routes, rows):
    """Every byte value in the encoding: all launches first, then one read of every status block."""
    enc = ENCODINGS[enc_name]
    cases = Cases()
    lut = None if enc.lut is None else torch.from_numpy(enc.lut).cuda()
    built = [build_chunk(enc_name, v, row_len) for v in BYTES]
    splits = [o.fastq_split(chunk) for chunk, _ in built]
    chunks = upload([chunk for chunk, _ in built], np.uint8)
    starts = upload([st[:, 1].astype(np.int64) for _, st, _ in splits], np.int64)
    lens = upload([ln[:, 1].astype(np.int32) for _, _, ln in splits], np.int32)
    offs = {}
    for span in (1, K, WINDOW):
        host = [out_offsets(ln[:, 1], span) for _, _, ln in splits]
        offs[span] = list(zip(upload([h[0] for h in host], np.int64), [h[1] for h in host]))
    for i, v in enumerate(BYTES):
        chunk, pos = built[i]
        want_bad = None if enc.alphabet[v] < 4 else (TARGET, pos)
        values = lambda k, window, chunk=chunk: oracle_values(chunk, enc, k, window)
        for name, route in routes.items():
            fused_count(cases, enc, lut, chunks[i], route, (enc_name, v, row_len, name), want_bad, values)
        if rows:
            row_entry_points(cases, enc, lut, chunks[i], starts[i], lens[i], {sp: o_[i] for sp, o_ in offs.items()},
                             (enc_name, v), want_bad, values)
    cases.verify()


@gpu
@pytest.mark.parametrize("enc_name", list(ENCODINGS))
def test_every_byte_on_every_route(enc_name):
    """Every fused-count route and the row entry points, rows of 150 bases and more."""
    run_cases(enc_name, ROW_LEN, ROUTES, rows=True)


@gpu
@pytest.mark.parametrize("enc_name", list(ENCODINGS))
def test_every_byte_in_a_deferred_row(enc_name):
    """A row longer than the warp-specialised count's row walk: the deferred rows_kernel encodes it."""
    run_cases(enc_name, LONG_ROW, {"ws": ROUTES["ws"]}, rows=False)


def test_placements_cover_every_unit_position():
    """CPU check of the placement rule: first, interior and last unit, all 16 positions in each, the byte in the row."""
    seen = set()
    for v in BYTES:
        for row_len in (ROW_LEN, LONG_ROW):
            r, length, pos = placement(v, row_len)
            assert 0 <= pos < length and length >= row_len
            unit = (r + pos) // 16
            last = (r + length - 1) // 16
            where = "first" if unit == 0 else "last" if unit == last else "interior"
            assert where != "interior" or 2 <= unit <= 6            # the steady state of the ws count
            seen.add((where, (r + pos) % 16))
    assert seen == {(w, p) for w in ("first", "interior", "last") for p in range(16)}
