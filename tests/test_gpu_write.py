"""Writers on the GPU: every byte the format kernel writes equals the NumPy writer oracle (tests/write_oracle.py), on
field views at unaligned starts with poison around every row, for any output slice; and the round trips through
bnp.open, including the reference's write scripts restated."""
import gzip
import io
import os

import numpy as np
import pytest
import torch

import bionumpy_b200 as bnp
from bionumpy_b200 import _native as nv
from bionumpy_b200 import ops
from bionumpy_b200.io import write as bw
from bionumpy_b200.io.ingest import _bgzf_blocks
from oracle import bnp_oracle as oracle

import write_oracle as wo
from helpers import make_fastq

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
DEV = "cuda"
POISON = 0xA5


def _place(rng, rows, pad=7):
    """A device byte buffer holding the rows at unaligned starts, poison before, between and after them."""
    starts, pos = [], int(rng.integers(1, 16))
    for r in rows:
        starts.append(pos)
        pos += len(r) + int(rng.integers(1, pad + 1))
    buf = np.full(pos + 16, POISON, dtype=np.uint8)
    for s, r in zip(starts, rows):
        buf[s:s + len(r)] = r
    return (torch.from_numpy(buf).to(DEV), torch.tensor(starts, dtype=torch.int64, device=DEV),
            torch.tensor([len(r) for r in rows], dtype=torch.int32, device=DEV))


def _rows(flat, lens):
    ends = np.cumsum(lens)
    return [flat[e - l:e] for e, l in zip(ends, lens)]


class Records:
    """Random records: names, sequences (text or codes) and qualities, host copies and device field views."""

    def __init__(self, rng, name_lens, seq_lens, alphabet="ACGT", codes=False):
        self.name_lens, self.seq_lens = np.asarray(name_lens), np.asarray(seq_lens)
        n = len(name_lens)
        self.names = rng.integers(33, 127, int(self.name_lens.sum()), dtype=np.uint8)
        letters = np.frombuffer(alphabet.encode(), dtype=np.uint8)
        code = rng.integers(0, len(alphabet), int(self.seq_lens.sum()))
        self.seqs = letters[code]
        self.quals = rng.integers(0, 94, int(self.seq_lens.sum())).astype(np.uint8)
        stored = code.astype(np.uint8) if codes else self.seqs
        self.lut = None
        if codes:
            t = np.zeros(256, dtype=np.uint8)
            t[:len(alphabet)] = letters
            self.lut = torch.from_numpy(t).to(DEV)
        self.fields = (_place(rng, _rows(self.names, self.name_lens)) + (None,),
                       _place(rng, _rows(stored, self.seq_lens)) + (self.lut,),
                       _place(rng, _rows(self.quals, self.seq_lens)) + (bw._lut("quality", None, torch.device(DEV)),))
        assert n == len(seq_lens)

    def text(self, fmt, width=1):
        if fmt == nv.FMT_FASTQ:
            return wo.fastq_text(self.names, self.name_lens, self.seqs, self.seq_lens, self.quals, self.seq_lens)
        if fmt == nv.FMT_FASTA:
            return wo.fasta_text(self.names, self.name_lens, self.seqs, self.seq_lens)
        return wo.multiline_fasta_text(self.names, self.name_lens, self.seqs, self.seq_lens, width)


def _format(rec, fmt, width=1, begin=0, end=None, out_shift=0):
    fields = rec.fields if fmt == nv.FMT_FASTQ else rec.fields[:2] + (None,)
    offsets, status = ops.format_offsets(fmt, width, fields)
    total = int(offsets[-1].item())
    end = total if end is None else end
    n = end - begin
    big = torch.full((n + 64,), POISON, dtype=torch.uint8, device=DEV)
    out = big[16 + out_shift:16 + out_shift + n]
    ops.format_records(fmt, width, fields, offsets, begin, end, out)
    host = big.cpu().numpy()
    outside = np.concatenate([host[:16 + out_shift], host[16 + out_shift + n:]])
    assert np.all(outside == POISON), "bytes written outside the slice"
    return host[16 + out_shift:16 + out_shift + n], offsets.cpu().numpy(), ops.read_status(status)


@pytest.mark.parametrize("fmt,width", [(nv.FMT_FASTQ, 1), (nv.FMT_FASTA, 1), (nv.FMT_FASTA_WRAPPED, 7)])
def test_slices_at_every_offset_mod_16_around_borders(fmt, width):
    rng = np.random.default_rng(fmt)
    rec = Records(rng, rng.integers(0, 40, 60), rng.integers(0, 90, 60))
    want = rec.text(fmt, width)
    full, offsets, _ = _format(rec, fmt, width)
    assert np.array_equal(full, want)
    assert offsets[-1] == want.size
    borders = sorted(set(offsets.tolist()) | set((offsets[:-1] + 1 + rec.name_lens).tolist()))
    for i, b in enumerate(borders[::3]):
        for d in range(-17, 18, 3):
            begin = int(np.clip(b + d, 0, want.size))
            end = int(min(want.size, begin + [1, 15, 16, 17, 33, 200][(i + d) % 6]))
            got, _, _ = _format(rec, fmt, width, begin, end, out_shift=(begin + d) % 16)
            assert np.array_equal(got, want[begin:end]), (begin, end)


@pytest.mark.parametrize("fmt", [nv.FMT_FASTQ, nv.FMT_FASTA, nv.FMT_FASTA_WRAPPED])
def test_empty_names_sequences_and_qualities(fmt):
    rng = np.random.default_rng(3)
    rec = Records(rng, [0, 0, 5, 0, 17, 0], [0, 3, 0, 40, 0, 0])
    got, _, _ = _format(rec, fmt, 4)
    assert np.array_equal(got, rec.text(fmt, 4))


@pytest.mark.parametrize("width", [1, 2, 15, 16, 17, 50, 60, 80, 4096])
def test_wrapped_widths(width):
    rng = np.random.default_rng(width)
    lens = [0, 1, width - 1, width, width + 1, 2 * width, 0, 2 * width + 3]
    rec = Records(rng, rng.integers(0, 20, len(lens)), lens)
    got, _, _ = _format(rec, nv.FMT_FASTA_WRAPPED, width)
    assert np.array_equal(got, rec.text(nv.FMT_FASTA_WRAPPED, width))


def test_long_rows_and_more_entries_than_one_grid():
    rng = np.random.default_rng(5)
    rec = Records(rng, [3, 70000, 2], [100000, 20, 50001])                  # rows longer than a 16 KiB output tile
    for fmt, width in ((nv.FMT_FASTQ, 1), (nv.FMT_FASTA, 1), (nv.FMT_FASTA_WRAPPED, 80)):
        got, _, _ = _format(rec, fmt, width)
        assert np.array_equal(got, rec.text(fmt, width))
    n = 250000                                                                 # ~25 MB: more tiles than the grid
    rec = Records(rng, rng.integers(0, 12, n), rng.integers(0, 40, n))
    got, _, _ = _format(rec, nv.FMT_FASTQ)
    assert np.array_equal(got, rec.text(nv.FMT_FASTQ))


@pytest.mark.parametrize("alphabet", ["ACGT", "ACTG", "ACDEFGHIKLMNPQRSTVWY*"])
def test_sequence_codes_and_bad_codes(alphabet):
    rng = np.random.default_rng(len(alphabet))
    rec = Records(rng, rng.integers(0, 9, 50), rng.integers(0, 70, 50), alphabet, codes=True)
    for fmt, width in ((nv.FMT_FASTQ, 1), (nv.FMT_FASTA_WRAPPED, 16)):
        got, _, st = _format(rec, fmt, width)
        assert st.bad_base() is None
        assert np.array_equal(got, rec.text(fmt, width))
    # an invalid code: its flat position in the sequence field
    seq_base, seq_starts, seq_lens, lut = rec.fields[1]
    flat_pos = int(rec.seq_lens[:30].sum()) + 5
    rows_before = np.cumsum(rec.seq_lens)
    row = int(np.searchsorted(rows_before, flat_pos, side="right"))
    pos = flat_pos - int(rows_before[row - 1] if row else 0)
    bad = seq_base.clone()
    bad[int(seq_starts[row]) + pos] = len(alphabet)
    bad[int(seq_starts[-1]) + int(rec.seq_lens[-1]) - 1] = 200 if rec.seq_lens[-1] else len(alphabet)
    enc = bnp.encodings.AlphabetEncoding(alphabet)
    seq = bnp.EncodedRaggedArray(bnp.EncodedArray(bad, enc), seq_lens, starts=seq_starts)
    names = bnp.EncodedRaggedArray(bnp.EncodedArray(rec.fields[0][0], bnp.BaseEncoding), rec.fields[0][2],
                                   starts=rec.fields[0][1])
    entries = bnp.SequenceEntry(names, seq)
    sink = io.BytesIO()
    w = bnp.NpBufferedWriter(sink, bnp.MultiLineFastaBuffer)
    with pytest.raises(bnp.EncodingError) as e:
        w.write(entries)
    assert e.value.offset == flat_pos
    w._sink.flush()
    assert sink.getvalue() == b""


def _read_all(path, **kw):
    return list(bnp.open(path, **kw).read_chunks())


def _concat_text(chunks, field):
    flat = [getattr(c, field).ravel() for c in chunks]
    return b"".join(bytes((f.raw() if hasattr(f, "raw") else f).cpu().numpy()) for f in flat)


def test_big_fastq_round_trips_plain_and_bgzf(tmp_path, big_fq_path, big_fq_bytes):
    for name in ("out.fq", "out.fq.gz"):
        path = tmp_path / name
        with bnp.open(path, "w") as f:
            for chunk in bnp.open(big_fq_path).read_chunks(min_chunk_size=100000):
                f.write(chunk)
        raw = path.read_bytes()
        text = gzip.decompress(raw) if name.endswith(".gz") else raw
        assert text == bytes(big_fq_bytes)
        if name.endswith(".gz"):
            assert _bgzf_blocks(memoryview(raw)) is not None
        a, b = _read_all(big_fq_path), _read_all(path)
        for field in ("name", "sequence", "quality"):
            assert _concat_text(a, field) == _concat_text(b, field)


def test_saccer3_written_at_width_50_is_the_file(tmp_path, monkeypatch):
    with gzip.open(os.path.join(GOLDEN, "sacCer3.fa.gz")) as f:
        data = f.read()
    monkeypatch.setattr(bnp.MultiLineFastaBuffer, "n_characters_per_line", 50)
    out = tmp_path / "y.fa"
    with bnp.open(out, "w") as f:
        f.write(bnp.open(os.path.join(GOLDEN, "sacCer3.fa.gz")))          # a reader, as convert_to_multiline.py
    assert out.read_bytes() == data


def test_synthetic_reads_written_back_byte_for_byte(tmp_path):
    n = 1000000
    chunk = ops.synth_fastq(n, device=DEV)
    buf = bnp.FastQBuffer.from_raw_buffer(chunk)
    entries = buf.get_data()
    assert entries.name[:1].tolist() == ["r0000000000"]
    text = bnp.FastQBuffer.from_data(entries)
    assert torch.equal(text.raw(), chunk)
    out = tmp_path / "s.fq"
    with bnp.open(out, "w") as f:
        f.write(entries)
    assert out.read_bytes() == bytes(chunk.cpu().numpy())


def test_crlf_input_is_written_with_lf(tmp_path):
    rng = np.random.default_rng(9)
    text = make_fastq(rng, 300, cr=True)
    src = tmp_path / "crlf.fq"
    src.write_bytes(bytes(text))
    out = tmp_path / "lf.fq"
    with bnp.open(out, "w") as f:
        f.write(bnp.open(src).read_chunks())
    assert out.read_bytes() == bytes(text).replace(b"\r\n", b"\n")


def test_write_in_several_slices(tmp_path, monkeypatch, big_fq_path, big_fq_bytes):
    monkeypatch.setattr(bw, "SLICE_BYTES", 4099)
    out = tmp_path / "sliced.fq.gz"
    with bnp.open(out, "w") as f:
        f.write(bnp.open(big_fq_path).read())
    assert gzip.decompress(out.read_bytes()) == bytes(big_fq_bytes)


def test_file_error_is_raised_by_a_later_call():
    class Broken(io.BytesIO):
        def write(self, b):
            raise OSError("disk full")

    w = bnp.NpBufferedWriter(Broken(), bnp.FastQBuffer)
    entries = bnp.SequenceEntryWithQuality(["a"], ["ACGT"], ["!!!!"])
    with pytest.raises(OSError):
        w.write(entries)
        w.write(entries)
        w.write(entries)
        w.close()


# ---- the reference's write scripts, restated -------------------------------------------------------------------------
def test_quality_filter_script(tmp_path, big_fq_path, big_fq_bytes):
    """scripts/fastq_filtering_example.py"""
    out = tmp_path / "filtered.fq.gz"
    with bnp.open(out, "w") as out_file:
        for reads in bnp.open(big_fq_path).read_chunks(min_chunk_size=200000):
            mask = (reads.quality.min(axis=-1) > 1) & (reads.quality.mean(axis=-1) > 10)
            out_file.write(reads[mask])
    n, nl, s, sl, q, ql = wo.read_fastq(big_fq_bytes)
    keep = np.array([len(row) > 0 and row.min() > 1 and row.mean() > 10 for row in _rows(q, ql)])
    sel = lambda flat, lens: (np.concatenate([r for r, k in zip(_rows(flat, lens), keep) if k] or [flat[:0]]), lens[keep])
    want = wo.fastq_text(*sel(n, nl), *sel(s, sl), *sel(q, ql))
    assert gzip.decompress(out.read_bytes()) == bytes(want)


def test_match_string_subsample_script(tmp_path, big_fq_path, big_fq_bytes):
    """scripts/subsample_reads_with_pattern_example.py: the reads that contain a pattern, to .fa.gz"""
    out = tmp_path / "hits.fa.gz"
    with bnp.open(out, "w") as f:
        for reads in bnp.open(big_fq_path).read_chunks():
            f.write(reads[np.sum(bnp.match_string(reads.sequence, "ACT"), axis=1) > 0])
    n, nl, s, sl, _, _ = wo.read_fastq(big_fq_bytes)
    keep = np.array([b"ACT" in bytes(r) for r in _rows(s, sl)])
    sel = lambda flat, lens: (np.concatenate([r for r, k in zip(_rows(flat, lens), keep) if k]), lens[keep])
    want = wo.multiline_fasta_text(*sel(n, nl), *sel(s, sl), 80)
    assert gzip.decompress(out.read_bytes()) == bytes(want)


def test_reverse_complement_script(tmp_path, big_fq_path, big_fq_bytes):
    """scripts/reverse_compliment_example.py with bnp.replace, and count_entries of input and output"""
    out = tmp_path / "rc.fq"
    with bnp.open(out, "w") as f:
        for chunk in bnp.open(big_fq_path).read_chunks():
            f.write(bnp.replace(chunk, sequence=bnp.get_reverse_complement(chunk.sequence)))
    assert bnp.count_entries(out) == bnp.count_entries(big_fq_path) == int(np.sum(big_fq_bytes == 10)) // 4
    n, nl, s, sl, q, ql = wo.read_fastq(big_fq_bytes)
    comp = oracle.complement_table()
    rc = np.concatenate([comp[r[::-1]] for r in _rows(s, sl)])
    assert out.read_bytes() == bytes(wo.fastq_text(n, nl, rc, sl, q, ql))


def test_streams_append_and_entries_from_lists(tmp_path):
    """test_io.py::test_write_dna_fastq, and appending chunks of a stream."""
    entry = bnp.SequenceEntryWithQuality(["name"], ["ACGT"], ["!!!!"])
    entry.sequence = bnp.as_encoded_array(entry.sequence, bnp.DNAEncoding)
    result = bnp.FastQBuffer.from_raw_buffer(bnp.FastQBuffer.from_data(entry)).get_data()
    assert result.sequence.tolist() == ["ACGT"] and result.quality.tolist() == [[0, 0, 0, 0]]
    path = tmp_path / "app.fq.gz"
    with bnp.open(path, "w") as f:
        f.write(entry)
    with bnp.open(path, "a") as f:
        f.write(x for x in [entry, entry[np.array([False])], bnp.SequenceEntryWithQuality(["n2"], ["GG"], ["II"])])
    assert gzip.decompress(path.read_bytes()) == b"@name\nACGT\n+\n!!!!\n@name\nACGT\n+\n!!!!\n@n2\nGG\n+\nII\n"
    with pytest.raises(ValueError):
        bnp.FastQBuffer.from_data(bnp.SequenceEntry(["a"], ["AC"]))
    with pytest.raises(ValueError):
        bnp.FastQBuffer.from_data(bnp.SequenceEntryWithQuality(["a", "b"], ["AC"], ["!!"]))
    with pytest.raises(TypeError):
        bnp.TwoLineFastaBuffer.from_data(bnp.SequenceEntry(["a"], bnp.get_kmers(bnp.as_encoded_array(["ACGT"], bnp.DNAEncoding), 2)))
    fa = bnp.TwoLineFastaBuffer.from_data(bnp.SequenceEntryWithQuality(["a"], ["AC"], ["!!"]))
    assert fa.to_string() == ">a\nAC\n"
    q = bnp.RaggedArray(torch.tensor([0, 222], dtype=torch.int64, device=DEV), [2])
    text = bnp.FastQBuffer.from_data(bnp.SequenceEntryWithQuality(["a"], ["AC"], q)).raw()
    assert bytes(text.cpu().numpy()) == b"@a\nAC\n+\n!\xff\n"
    with pytest.raises(ValueError):
        bnp.FastQBuffer.from_data(bnp.SequenceEntryWithQuality(
            ["a"], ["AC"], bnp.RaggedArray(torch.tensor([0, 223], device=DEV), [2])))


@pytest.mark.parametrize("fmt,width", [(nv.FMT_FASTA, 1), (nv.FMT_FASTA_WRAPPED, 60)])
def test_bad_code_reported_at_its_exact_position(fmt, width):
    """One bad code at every position of a row, inside and across the 16-byte units the kernel gathers whole."""
    rng = np.random.default_rng(11)
    rec = Records(rng, [5, 3, 9, 1], [64, 70, 64, 3], "ACGT", codes=True)
    seq_base, seq_starts, seq_lens, lut = rec.fields[1]
    for pos in range(64):
        bad = seq_base.clone()
        bad[int(seq_starts[2]) + pos] = 4
        fields = (rec.fields[0], (bad, seq_starts, seq_lens, lut), None)
        _, status = ops.format_offsets(fmt, width, fields)
        assert ops.read_status(status).bad_base() == (2, pos), pos
