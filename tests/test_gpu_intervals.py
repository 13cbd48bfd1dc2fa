"""BED parsing, contig lookup and interval sequences on the GPU (csrc/interval_kernels.cu) against the NumPy restatement
of the reference (tests/interval_oracle.py), value for value and byte for byte.

Chunks are views at byte offsets 0..15 of an allocation with poison after the view, so a read past the chunk changes a
value or reports a fault."""
import gzip
import os
import warnings

import numpy as np
import pytest
import torch

import bionumpy_b200 as bnp
from bionumpy_b200 import _native as nv
from bionumpy_b200.io import Bed6Buffer, BedBuffer, FormatException
from bionumpy_b200.sequence import get_sequences, get_strand_specific_sequences

import interval_oracle as io_
import motif_oracle as mo

gpu = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
POISON = b"\t7\t-\r\n9"


def _view(text, off):
    """``text`` on the device at byte offset ``off`` of its allocation, poison after it."""
    buf = torch.frombuffer(bytearray(b"x" * off + text + POISON * 4), dtype=torch.uint8).cuda()
    return buf[off:off + len(text)]


def _text_rows(field):
    return [bytes(r.cpu().numpy()) for r in field.raw()]


def _assert_columns(buf, cols, kinds):
    for i, (kind, want) in enumerate(zip(kinds, cols)):
        got = buf.get_field_by_number(i)
        if kind == io_.TEXT:
            assert _text_rows(got) == want, i
        elif kind == io_.STRAND:
            assert got.raw().cpu().numpy().tolist() == want.tolist(), i
        else:
            assert got.cpu().numpy().tolist() == want.tolist(), i


def _parse(text, buffer_type, kinds, off=0):
    size, cols = io_.parse_delimited(text, kinds)
    buf = buffer_type.from_raw_buffer(_view(text, off))
    assert buf.size == size and buf.n_lines == text[:size].count(b"\n") == len(buf.get_data())
    _assert_columns(buf, cols, kinds)
    return buf


def _random_bed6(rng, n, crlf=False):
    lines = []
    for _ in range(n):
        chrom = b"chr" + bytes(rng.choice(list(b"0123456789XYMabc_"), rng.integers(0, 30)).tolist())
        start = int(rng.integers(0, 10 ** int(rng.integers(1, 19))))
        stop = int(rng.integers(0, 10 ** int(rng.integers(1, 19))))
        name = bytes(rng.choice(list(b"abcdefgh.-_"), rng.integers(0, 40)).tolist())
        score = b"." if rng.random() < 0.3 else str(int(rng.integers(-10 ** 6, 10 ** 6))).encode()
        strand = bytes([b"+-."[rng.integers(0, 3)]])
        lines.append(b"\t".join([chrom, str(start).encode(), str(stop).encode(), name, score, strand]) +
                     (b"\r\n" if crlf else b"\n"))
    return b"".join(lines)


@gpu
@pytest.mark.parametrize("off", range(16))
def test_parse_at_every_view_offset(off):
    rng = np.random.default_rng(off)
    _parse(_random_bed6(rng, 300), Bed6Buffer, io_.BED6, off)
    _parse(_random_bed6(rng, 50) + b"chr1\t5\t", Bed6Buffer, io_.BED6, off)        # an incomplete last line is cut


@gpu
def test_fields_around_unit_edges():
    """Lines of 6..70 bytes whose tabs fall on every byte of a 16-byte unit, staged (short lines) or not (long)."""
    lines = []
    for a in range(1, 33):
        for b in range(1, 19):
            lines.append(b"c" * a + b"\t" + b"1" * b + b"\t" + b"2" * ((a + b) % 18 + 1) + b"\n")
    text = b"".join(lines)
    for off in (0, 1, 7, 15):
        _parse(text, BedBuffer, io_.BED, off)
    long = b"".join(b"c" * 300 + b"\t1\t" + b"9" * 18 + b"\n" for _ in range(200))   # 128 lines > the 16 KiB stage
    _parse(long, BedBuffer, io_.BED)


@gpu
def test_integers_of_every_width_and_sign():
    rng = np.random.default_rng(3)
    lines = []
    for d in range(1, 19):
        for sign in (b"", b"-", b"+"):
            for _ in range(8):
                v = b"".join(bytes([48 + int(x)]) for x in rng.integers(0, 10, d))
                lines.append(b"chr\t" + sign + v + b"\t" + v + b"\t.\t" + sign + v + b"\t+\n")
    _parse(b"".join(lines), Bed6Buffer, io_.BED6)


@gpu
def test_dot_scores_and_carriage_returns():
    text = b"chr1\t1\t3\t.\t.\t-\nchr1\t40\t60\tx\t7\t+\nchr20\t400\t600\t.\t.\t.\n"
    buf = _parse(text, Bed6Buffer, io_.BED6)
    assert buf.get_data().score.cpu().tolist() == [0, 7, 0]
    _parse(_random_bed6(np.random.default_rng(5), 200, crlf=True), Bed6Buffer, io_.BED6)
    buf = _parse(b"chr1\t1\t2\r\nchr2\t3\t4\n", BedBuffer, io_.BED)            # test_io.py::test_carriage_return_bed
    assert buf.get_data().stop.cpu().tolist() == [2, 4]


def _faulty(where, what, n=40):
    lines = [b"chr%d\t%d\t%d\tn\t%d\t+\n" % (i % 3, i, i + 10, i) for i in range(n)]
    i = {"first": 0, "interior": n // 2, "last": n - 1}[where]
    lines[i] = {"tabs": b"chr1\t1\t2\tn\t0\n", "extra": b"chr1\t1\t2\tn\t0\t+\tx\n", "digit": b"chr1\t1\t2x\tn\t0\t+\n",
                "sign": b"chr1\t-\t2\tn\t0\t+\n", "wide": b"chr1\t1\t1234567890123456789\tn\t0\t+\n",
                "strand": b"chr1\t1\t2\tn\t0\tx\n", "score": b"chr1\t1\t2\tn\t..\t+\n"}[what]
    return b"".join(lines)


@gpu
@pytest.mark.parametrize("where", ["first", "interior", "last"])
@pytest.mark.parametrize("what", ["tabs", "extra", "digit", "sign", "wide", "strand", "score"])
def test_faults_raise_the_reference_line(where, what):
    text = _faulty(where, what)
    with pytest.raises(io_.Fault) as want:
        io_.parse_delimited(text, io_.BED6)
    with pytest.raises(FormatException) as got:
        Bed6Buffer.from_raw_buffer(_view(text, 3))
    assert got.value.line_number == want.value.line


@gpu
def test_too_few_columns_for_the_record():
    with pytest.raises(FormatException) as e:
        Bed6Buffer.from_raw_buffer(_view(b"chr1\t1\t2\nchr1\t3\t4\n", 0))
    assert e.value.line_number == 0


@gpu
def test_every_chunk_size_carries_entries(tmp_path):
    text = b"#comment one\n#two\n" + _random_bed6(np.random.default_rng(9), 6)
    body = text[text.index(b"chr"):]
    want = io_.read_delimited(body, io_.BED6, 1 << 20)
    path = tmp_path / "x.bed"
    path.write_bytes(text)
    for size in range(1, len(body) + 1):
        with bnp.open(str(path), buffer_type=Bed6Buffer) as f:
            chunks = list(f.read_chunks(min_chunk_size=size))
        got_start = torch.cat([c.start for c in chunks]).cpu().numpy()
        assert got_start.tolist() == want[1].tolist(), size
        assert [r for c in chunks for r in _text_rows(c.name)] == want[3], size
        assert np.concatenate([c.strand.raw().cpu().numpy() for c in chunks]).tolist() == want[5].tolist(), size


@gpu
@pytest.mark.parametrize("size", [200, 333, 4096])
def test_reader_fault_line_is_global(tmp_path, size):
    """test_io_exceptions.py::test_npdataclass_raises_format_exception_bed: line 4 * 100 + 1."""
    path = tmp_path / "bad.bed"
    path.write_bytes(b"chr1\t10\t20\nchr2\t20\t30\nchr1\t10\t20\nchr2\t20\t30\n" * 100 + b"chr1\t10\t20\nchr2\t10\ttwenty\n")
    with pytest.raises(FormatException) as e:
        for chunk in bnp.open(str(path)).read_chunks(size):
            chunk.stop
    assert e.value.line_number == 401


@gpu
def test_ctcf_whole_file():
    data = gzip.open(os.path.join(GOLDEN, "ctcf.bed.gz")).read()
    chrom, start, stop = io_.read_delimited(data, io_.BED, 1 << 30)
    peaks = bnp.open(os.path.join(GOLDEN, "ctcf.bed.gz")).read()
    assert isinstance(peaks, bnp.Interval) and len(peaks) == 44722
    assert peaks.start.cpu().numpy().tolist() == start.tolist() and peaks.stop.cpu().numpy().tolist() == stop.tolist()
    assert _text_rows(peaks.chromosome) == chrom


@gpu
def test_ten_million_lines():
    names = ["chr%d" % i for i in range(1, 23)] + ["chrX", "chrUn_gl000220"]
    text, ci, start, stop = io_.synthetic_bed(10_000_000, names, seed=1)
    buf = BedBuffer.from_raw_buffer(torch.frombuffer(bytearray(text), dtype=torch.uint8).cuda())
    assert buf.n_lines == 10_000_000 and buf.size == len(text)
    d = buf.get_data()
    assert torch.equal(d.start.cpu(), torch.from_numpy(start)) and torch.equal(d.stop.cpu(), torch.from_numpy(stop))
    lens = np.array([len(n) for n in names])[ci]
    assert np.array_equal(d.chromosome.lengths.cpu().numpy(), lens)
    starts = d.chromosome._starts.cpu().numpy()
    head = np.frombuffer(text, dtype=np.uint8)[starts]                      # each view starts on its "chr"
    assert np.all(head == ord("c"))
    # every name byte, checked by its index: the 5th byte of each name
    fifth = np.frombuffer(text, dtype=np.uint8)[starts + 4]
    name5 = np.array([ord(n[4]) if len(n) > 4 else ord("\t") for n in names])[ci]
    assert np.array_equal(fifth, name5)
    # the first 10 000 lines through the oracle itself
    cut = text[:int(np.flatnonzero(np.frombuffer(text[:1 << 20], dtype=np.uint8) == 10)[9999]) + 1]
    _, (c2, s2, e2) = io_.parse_delimited(cut, io_.BED)
    assert s2.tolist() == start[:10000].tolist() and e2.tolist() == stop[:10000].tolist()
    assert c2 == [names[i].encode() for i in ci[:10000]]


# ---- lookup and gather ----------------------------------------------------------------------------------------------

def _sac_cer3(tmp_path):
    raw = gzip.open(os.path.join(GOLDEN, "sacCer3.fa.gz")).read()
    path = tmp_path / "sacCer3.fa"
    path.write_bytes(raw)
    fa = bnp.open_indexed(str(path))
    index = {k: v for k, v in fa._index.items()}
    return raw, index, fa


def _oracle_rows(raw, index, chroms, starts, stops):
    flat, lens = io_.interval_sequences(raw, index, chroms, starts, stops)
    return flat, lens


def _check(fa, raw, index, chroms, starts, stops):
    got = fa.get_interval_sequences(bnp.Interval(list(chroms), list(starts), list(stops)))
    flat, lens = _oracle_rows(raw, index, chroms, starts, stops)
    assert got.lengths.cpu().numpy().tolist() == lens.tolist()
    assert np.array_equal(got.ravel().raw().cpu().numpy(), flat)
    # the host list path gives the same bytes
    host = fa.get_interval_sequences(list(zip(chroms, starts, stops)))
    assert np.array_equal(host.ravel().raw().cpu().numpy(), flat)


@gpu
def test_small_genome_golden():
    fa = bnp.open_indexed(os.path.join(GOLDEN, "small_genome.fa"))
    raw = open(os.path.join(GOLDEN, "small_genome.fa"), "rb").read()
    tuples = [("1", 10, 20), ("2", 11, 50), ("1", 5, 10), ("3", 10, 110), ("1", 80, 250)]
    _check(fa, raw, fa._index, *map(list, zip(*tuples)))
    seqs = fa.get_interval_sequences(bnp.Interval.from_entry_tuples(tuples))
    assert seqs.lengths.cpu().tolist() == [10, 39, 5, 100, 170]


@gpu
def test_edges_of_every_contig(tmp_path):
    raw, index, fa = _sac_cer3(tmp_path)
    chroms, starts, stops = [], [], []
    for name, idx in index.items():
        L, c = idx["rlen"], idx["lenc"]
        for a, b in ((0, 0), (0, 1), (0, L), (L - 1, L), (L, L), (c - 1, c + 1), (c, 2 * c), (c - 1, 3 * c + 1),
                     (L - c - 1, L), (5, 5 + 16), (c - 8, c + 8), (L - 17, L - 1)):
            chroms.append(name), starts.append(a), stops.append(b)
        for k in range(1, min(L // c, 40)):                                   # intervals on every line boundary
            for a, b in ((k * c - 1, k * c), (k * c, k * c + 1), (k * c - 16, k * c + 16), (k * c - 3, k * c + 100)):
                chroms.append(name), starts.append(a), stops.append(min(b, L))
    _check(fa, raw, index, chroms, starts, stops)


@gpu
def test_bad_intervals_raise(tmp_path):
    raw, index, fa = _sac_cer3(tmp_path)
    name = next(iter(index))
    L = index[name]["rlen"]
    for a, b in ((0, L + 1), (-1, 5), (10, 9)):
        with pytest.raises(ValueError):
            fa.get_interval_sequences(bnp.Interval([name, name], [0, a], [10, b]))
    with pytest.raises(KeyError, match="chrNope"):
        fa.get_interval_sequences(bnp.Interval([name, "chrNope"], [0, 0], [10, 10]))


@gpu
def test_names_that_are_prefixes_of_each_other(tmp_path):
    names = ["chr1", "chr10", "chr1_alt", "c", "chr11", "chr1\x7f", "b", "chr100"]
    rng = np.random.default_rng(2)
    text, contigs = b"", {}
    for i, n in enumerate(names):
        seq = bytes(rng.choice(list(b"ACGTacgtN"), 50 + 37 * i).tolist())
        contigs[n] = seq
        text += b">" + n.encode() + b" desc\n" + b"\n".join(seq[j:j + 13] for j in range(0, len(seq), 13)) + b"\n"
    path = tmp_path / "p.fa"
    path.write_bytes(text)
    fa = bnp.open_indexed(str(path))
    chroms = [names[int(i)] for i in rng.integers(0, len(names), 500)]
    starts = [int(rng.integers(0, 40)) for _ in chroms]
    stops = [s + int(rng.integers(0, 10)) for s in starts]
    got = fa.get_interval_sequences(bnp.Interval(chroms, starts, stops))
    want = b"".join(contigs[c][a:b] for c, a, b in zip(chroms, starts, stops))
    assert bytes(got.ravel().raw().cpu().numpy()) == want
    for unknown in ("chr", "chr1_", "chr1000", "d", "chr10\x00"):
        with pytest.raises(KeyError):
            fa.get_interval_sequences(bnp.Interval(["chr1", unknown], [0, 0], [1, 1]))


@gpu
def test_a_million_random_intervals(tmp_path):
    raw, index, fa = _sac_cer3(tmp_path)
    names = list(index)
    rng = np.random.default_rng(7)
    n = 1_000_000
    ci = rng.integers(0, len(names), n)
    rlen = np.array([index[k]["rlen"] for k in names])[ci]
    width = rng.integers(0, 300, n)
    starts = (rng.random(n) * (rlen - width + 1)).astype(np.int64)
    stops = starts + width
    chroms = [names[i] for i in ci]
    got = fa.get_interval_sequences(bnp.Interval(chroms, starts, stops))
    # every byte against the contigs without line ends, and the first 20 000 through the seek-and-delete loop itself
    contig = {}
    for k in names:
        i = index[k]
        rows = (i["rlen"] + i["lenc"] - 1) // i["lenc"]
        body = np.frombuffer(raw, dtype=np.uint8)[i["offset"]: i["offset"] + rows * i["lenb"]]
        contig[k] = np.delete(body, np.arange(i["lenc"], body.size, i["lenb"]))[:i["rlen"]]
    flat_all = np.concatenate([contig[k] for k in names])
    base = np.concatenate([[0], np.cumsum([index[k]["rlen"] for k in names])])[ci]
    idx = np.repeat(base + starts - np.concatenate([[0], np.cumsum(width)])[:-1], width) + np.arange(width.sum())
    assert np.array_equal(got.lengths.cpu().numpy(), width)
    assert np.array_equal(got.ravel().raw().cpu().numpy(), flat_all[idx])
    m = 20_000
    flat, lens = _oracle_rows(raw, index, chroms[:m], starts[:m].tolist(), stops[:m].tolist())
    assert np.array_equal(got.ravel().raw().cpu().numpy()[:flat.size], flat)


@gpu
@pytest.mark.parametrize("encoded", [False, True])
def test_strand_specific_sequences(encoded):
    rng = np.random.default_rng(11 + encoded)
    text = bytes(rng.choice(list(b"ACGTNacgtnRY"), 5000).tolist())
    if encoded:
        text = bytes(rng.choice(list(b"ACGT"), 5000).tolist())
        seq = bnp.as_encoded_array(text.decode(), bnp.DNAEncoding)
        host = np.array(["ACGT".index(chr(c)) for c in text], dtype=np.uint8)
        alphabet = "ACGT"
    else:
        seq = bnp.as_encoded_array(text.decode())
        host, alphabet = np.frombuffer(text, dtype=np.uint8), None
    n = 2000
    starts = rng.integers(0, 4900, n)
    stops = starts + rng.integers(0, 100, n)
    strands = ["+-."[int(s)] for s in rng.integers(0, 3, n)]
    iv = bnp.datatypes.StrandedInterval(["c"] * n, starts, stops, strands)
    want = io_.strand_specific_sequences(host, starts, stops, strands, alphabet)
    got = get_strand_specific_sequences(seq, iv)
    assert got.encoding == seq.encoding
    assert got.lengths.cpu().numpy().tolist() == [len(w) for w in want]
    assert np.array_equal(got.ravel().raw().cpu().numpy(), np.concatenate(want))
    plain = get_sequences(seq, iv)
    assert np.array_equal(plain.ravel().raw().cpu().numpy(), np.concatenate([host[a:b] for a, b in zip(starts, stops)]))
    # the reference's own golden (test_dna.py::test_strand_specific_sequences)
    dna = bnp.as_encoded_array("ACGTACGTACGT", bnp.DNAEncoding)
    res = get_strand_specific_sequences(dna, bnp.datatypes.Bed6(["chr1", "chr1"], [1, 4], [3, 7], [".", "."], [".", "."],
                                                                ["+", "-"]))
    assert res.tolist() == ["CG", "CGT"]
    with pytest.raises(ValueError):
        get_sequences(seq, bnp.Interval(["c"], [4990], [5001]))


def _intervals_for(fa, n, seed):
    names = list(fa._index)
    rng = np.random.default_rng(seed)
    ci = rng.integers(0, len(names), n)
    starts = rng.integers(0, 1000, n)
    return bnp.Interval([names[i] for i in ci], starts, starts + 100)


@gpu
def test_one_synchronisation_and_constant_launches(tmp_path):
    _, _, fa = _sac_cer3(tmp_path)
    lib = nv.load_library()
    fa.get_interval_sequences(_intervals_for(fa, 10, 0))                 # builds the name table
    launches = []
    for n in (10, 1_000_000):
        iv = _intervals_for(fa, n, n)
        torch.cuda.synchronize()
        before = lib.bnpk_launch_count()
        torch.cuda.set_sync_debug_mode("warn")
        try:
            with warnings.catch_warnings(record=True) as caught:
                warnings.simplefilter("always")
                out = fa.get_interval_sequences(iv)
        finally:
            torch.cuda.set_sync_debug_mode(0)
        launches.append(lib.bnpk_launch_count() - before)
        syncs = [w for w in caught if "synchroniz" in str(w.message)]
        assert len(syncs) == 1, [str(w.message) for w in caught]
        assert out.lengths.numel() == n
    assert launches[0] == launches[1], launches


@gpu
def test_manuscript_chain(tmp_path):
    """scripts/manuscript_code2.py on sacCer3 with a synthetic peak BED and MA0080.1."""
    raw, index, fa = _sac_cer3(tmp_path)
    names = list(index)
    rng = np.random.default_rng(4)
    n = 5000
    ci = rng.integers(0, len(names), n)
    rlen = np.array([index[k]["rlen"] for k in names])[ci]
    mid = (rng.random(n) * (rlen - 400)).astype(np.int64) + 200
    half = rng.integers(20, 150, n)
    lines = [b"%s\t%d\t%d\tpeak%d\t%d\t.\n" % (names[c].encode(), m - h, m + h, i, i % 1000)
             for i, (c, m, h) in enumerate(zip(ci, mid, half))]
    bed = tmp_path / "peaks.bed"
    bed.write_bytes(b"".join(lines))
    pwm = bnp.io.read_motif(os.path.join(GOLDEN, "MA0080.1.jaspar"))

    peaks = bnp.open(str(bed)).read()
    midpoints = (peaks.start + peaks.stop) // 2
    peaks.start = midpoints - 50
    peaks.stop = midpoints + 50
    seqs = bnp.open_indexed(str(tmp_path / "sacCer3.fa")).get_interval_sequences(peaks)
    hits = bnp.get_motif_scores(seqs, pwm) > np.log(4)
    got = np.mean(hits, axis=0)

    chrom, start, stop = io_.parse_delimited(b"".join(lines), io_.BED)[1]
    m2 = (start + stop) // 2
    flat, lens = io_.interval_sequences(raw, index, [c.decode() for c in chrom], (m2 - 50).tolist(), (m2 + 50).tolist())
    codes, bad = mo.encode([bytes(flat)], "ACGT")
    assert bad is None
    scores, s_lens = mo.motif_scores(codes, lens, pwm._matrix)
    want_hits = (scores > np.log(4)).reshape(n, -1)
    assert np.array_equal(hits.ravel().cpu().numpy(), want_hits.ravel())
    got = torch.as_tensor(got).cpu().numpy()                    # summed in another order than NumPy's: last bits
    assert np.array_equal(np.rint(got * n), want_hits.sum(axis=0)) and np.allclose(got, want_hits.mean(axis=0), 0, 1e-15)


@gpu
def test_mean_axis0_needs_equal_rows():
    r = bnp.RaggedArray(torch.arange(6, device="cuda"), [3, 3])
    assert r.mean(axis=0).cpu().tolist() == [1.5, 2.5, 3.5]
    with pytest.raises(NotImplementedError):
        bnp.RaggedArray(torch.arange(6, device="cuda"), [2, 4]).mean(axis=0)


@gpu
def test_records_and_writing(tmp_path):
    iv = bnp.Interval(["chr1"], [2], [100])
    assert iv.start.is_cuda and iv.chromosome.tolist() == ["chr1"]
    iv.start = iv.start + 1
    assert iv.start.cpu().tolist() == [3]
    sub = bnp.replace(iv, stop=torch.tensor([50], device="cuda"))
    assert sub.stop.cpu().tolist() == [50] and sub.start.cpu().tolist() == [3]
    b6 = bnp.Bed6.from_entry_tuples([("chr1", 1, 3, ".", 0, "-"), ("chr2", 4, 9, "x", 5, "+")])
    assert b6[torch.tensor([True, False], device="cuda")].strand.raw().cpu().tolist() == [1]
    with pytest.raises(NotImplementedError):
        bnp.open(str(tmp_path / "out.bed"), "w")


@gpu
def test_reference_example_files():
    """example_data/small_interval.bed on small_genome.fa and alignments.bed as Bed6, through bnp.open."""
    fa_path = os.path.join(GOLDEN, "small_genome.fa")
    raw = open(fa_path, "rb").read()
    text = open(os.path.join(GOLDEN, "small_interval.bed"), "rb").read()
    chrom, start, stop = io_.parse_delimited(text, io_.BED)[1]
    peaks = bnp.open(os.path.join(GOLDEN, "small_interval.bed")).read()
    assert _text_rows(peaks.chromosome) == chrom and peaks.stop.cpu().tolist() == stop.tolist()
    fa = bnp.open_indexed(fa_path)
    got = fa.get_interval_sequences(peaks)
    flat, lens = io_.interval_sequences(raw, fa._index, [c.decode() for c in chrom], start.tolist(), stop.tolist())
    assert got.lengths.cpu().tolist() == lens.tolist()
    assert np.array_equal(got.ravel().raw().cpu().numpy(), flat)
    text = open(os.path.join(GOLDEN, "alignments.bed"), "rb").read()
    want = io_.parse_delimited(text, io_.BED6)[1]
    with bnp.open(os.path.join(GOLDEN, "alignments.bed"), buffer_type=Bed6Buffer) as f:
        reads = f.read()
    assert isinstance(reads, bnp.Bed6)
    assert _text_rows(reads.chromosome) == want[0] and reads.start.cpu().tolist() == want[1].tolist()
    assert reads.score.cpu().tolist() == want[4].tolist() and reads.strand.raw().cpu().tolist() == want[5].tolist()


@gpu
def test_dispatcher_ops_match_the_ctypes_path():
    from bionumpy_b200 import ops, torch_ops
    top = torch_ops.load()
    text = _random_bed6(np.random.default_rng(21), 500)
    chunk = _view(text, 5)
    starts, lens, _ = ops.line_split(chunk, 1, 0, 0, ord("#"), False, 0, max_rows=text.count(b"\n"))
    kinds = list(Bed6Buffer._kinds)
    want, _ = ops.delimited_columns(chunk, starts, lens, kinds)
    values, text_lens, status = top.delimited_columns(chunk, starts, lens, kinds)
    assert int(status[nv.ST_BAD_BASE]) == nv.INT64_MAX
    for kind, w, v, tl in zip(kinds, want, values, text_lens):
        if kind == nv.COL_TEXT:
            assert torch.equal(v, w[0]) and torch.equal(tl, w[1])
        else:
            assert torch.equal(v, w)
    fa = bnp.open_indexed(os.path.join(GOLDEN, "small_genome.fa"))
    _, names, name_offsets, contigs = fa._name_table()
    iv = bnp.Interval(["1", "3", "0", "2"], [0, 79, 5, 100], [80, 81, 5, 300])
    from bionumpy_b200.rows import RowView
    rows = RowView(iv.chromosome)
    ids, st = top.name_lookup(rows.base, rows.starts, rows.lens, names, name_offsets)
    assert int(st[nv.ST_BAD_BASE]) == nv.INT64_MAX
    assert torch.equal(ids, ops.name_lookup(rows.base, rows.starts, rows.lens, names, name_offsets)[0])
    row_lens, st = top.interval_check(fa._file, iv.start, iv.stop, ids, list(contigs))
    assert int(st[nv.ST_BAD_BASE]) == nv.INT64_MAX and row_lens.cpu().tolist() == [80, 2, 0, 200]
    offsets = ops.row_offsets(row_lens)
    out = top.interval_copy(fa._file, iv.start, iv.stop, ids, list(contigs), None, None, offsets, 282)
    assert torch.equal(out, fa.get_interval_sequences(iv).ravel().raw())
    bad = bnp.Interval(["1"], [0], [601])                               # contig "1" has 600 bases
    _, st = top.interval_check(fa._file, bad.start, bad.stop, ids[:1], list(contigs))
    assert int(st[nv.ST_BAD_BASE]) == 0
