"""BED and bedGraph text from device columns (bnpk_delimited_offsets / bnpk_delimited_format) and the writer around
them, against tests/delimited_write_oracle.py."""
import gzip
import os

import numpy as np
import pytest
import torch

import bionumpy_b200 as bnp
from bionumpy_b200 import _native as nv
from bionumpy_b200 import ops, torch_ops
from bionumpy_b200.io import write as bw
from bionumpy_b200.io.delimited import DelimitedText

import delimited_write_oracle as wo
import interval_oracle as io_

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
I64 = np.iinfo(np.int64)


def _digit_borders():
    out = [0, I64.max, I64.min, I64.min + 1]
    for d in range(1, 19):
        p = 10 ** d
        out += [p - 1, p, p + 1, -(p - 1), -p, -(p + 1)]
    return np.array(out, dtype=np.int64)


def _text(entries):
    return bytes(bnp.io.BedBuffer.from_data(entries).raw().cpu().numpy())


def _bed6(rng, n, names=("chr1", "chr10", "", "chrUn_KI270302v1")):
    chroms = [names[i] for i in rng.integers(0, len(names), n)]
    start = rng.integers(-10 ** 12, 10 ** 12, n)
    stop = rng.integers(0, 10 ** 6, n)
    name = ["".join("ab"[j] for j in rng.integers(0, 2, k)) for k in rng.integers(0, 12, n)]
    score = rng.integers(-5, 1000, n)
    strand = rng.integers(0, 3, n)
    entries = bnp.Bed6(chroms, start, stop, name, score, "".join("+-."[s] for s in strand))
    want = wo.dump_lines([("text", chroms), ("int", start), ("int", stop), ("text", name), ("int", score),
                          ("strand", strand)])
    return entries, want


def test_every_column_kind():
    entries, want = _bed6(np.random.default_rng(1), 3000)
    assert _text(entries) == want
    assert bytes(bnp.io.Bed6Buffer.from_data(entries).raw().cpu().numpy()) == want
    iv = bnp.Interval(["chr1", "chr10"], [1, 2], [3, 4])
    assert _text(iv) == b"chr1\t1\t3\nchr10\t2\t4\n"
    st = bnp.StrandedInterval(["a", "b", "c"], [0, 1, 2], [5, 6, 7], "+-.")
    assert _text(st) == b"a\t0\t5\t+\nb\t1\t6\t-\nc\t2\t7\t.\n"
    bg = bnp.BedGraph(["x", "y"], [0, 3], [3, 9], np.array([-4, 7], dtype=np.int16))
    assert bytes(bnp.io.BdgBuffer.from_data(bg).raw().cpu().numpy()) == b"x\t0\t3\t-4\ny\t3\t9\t7\n"


def test_integers_at_every_digit_count():
    v = _digit_borders()
    iv = bnp.Interval(["c"] * v.size, v, v[::-1].copy())
    assert _text(iv) == wo.dump_lines(wo.bed_columns(["c"] * v.size, v, v[::-1]))
    # the dispatcher ops give the same bytes
    cols = [(nv.COL_INT, torch.from_numpy(v).cuda())]
    offs, _ = torch_ops.load().delimited_offsets([cols[0][1]], [nv.COL_INT])
    out = torch_ops.load().delimited_format([cols[0][1]], [nv.COL_INT], offs, 0, int(offs[-1]))
    assert bytes(out.cpu().numpy()) == wo.dump_lines([("int", v)])


def test_empty_text_fields_and_names_of_different_lengths():
    chroms = ["chr1", "chr10", "", "c", "chr1" * 40, ""]
    iv = bnp.Interval(chroms, list(range(6)), list(range(1, 7)))
    assert _text(iv) == wo.dump_lines(wo.bed_columns(chroms, range(6), range(1, 7)))


def test_bad_strand_codes_and_mismatched_fields():
    codes = torch.tensor([0, 1, 2, 3, 7], dtype=torch.uint8, device="cuda")
    ints = torch.arange(5, dtype=torch.int64, device="cuda")
    offs, status = ops.delimited_offsets([(nv.COL_INT, ints), (nv.COL_STRAND, codes)])
    fault = int(status[nv.ST_BAD_BASE].item())
    assert fault == (3 << 8 | 1 << 3 | nv.BAD_STRAND)
    assert bytes(ops.delimited_format([(nv.COL_INT, ints), (nv.COL_STRAND, codes)], offs).cpu().numpy()) == \
        b"0\t+\n1\t-\n2\t.\n3\t.\n4\t.\n"
    st = bnp.StrandedInterval(["a"] * 2, [0, 1], [1, 2], "+-")
    st.strand = bnp.EncodedArray(torch.tensor([0, 9], dtype=torch.uint8, device="cuda"), bnp.StrandEncoding)
    with pytest.raises(ValueError, match="line 1"):
        _text(st)
    with pytest.raises(ValueError, match="differ in length"):
        ops.delimited_offsets([(nv.COL_INT, ints), (nv.COL_INT, ints[:3])])
    with pytest.raises(ValueError):
        _text(bnp.Interval(["a", "b"], [0, 1], [1]))
    with pytest.raises(TypeError):
        bnp.io.BdgBuffer.from_data(bnp.BedGraph(["x"], [0], [3], np.array([0.5])))
    with pytest.raises(TypeError):
        _text(bnp.SequenceEntry(["a"], ["ACGT"]))
    with pytest.raises(NotImplementedError):
        bnp.io.BdgBuffer.from_raw_buffer(bnp.as_encoded_array("x\t0\t1\t0.5\n"))


def test_output_windows_cut_lines_at_every_offset():
    """Slices [a, b) of the text at every offset of a few lines, into outputs at every alignment."""
    entries, want = _bed6(np.random.default_rng(2), 40)
    text = DelimitedText(entries)
    assert text.size == len(want)
    store = torch.empty(len(want) + 32, dtype=torch.uint8, device="cuda")
    for a in range(0, len(want), 7):
        for b in (a, a + 1, a + 13, len(want)):
            b = min(b, len(want))
            for shift in (0, 1, 15):
                out = store[shift:shift + b - a]
                text.slice(a, b, out)
                assert bytes(out.cpu().numpy()) == want[a:b], (a, b, shift)


def test_windows_and_lines_past_one_window():
    """Lines longer than a CTA's 16 KiB window and windows full of short lines."""
    rng = np.random.default_rng(3)
    names = ["x" * int(k) for k in rng.integers(0, 40000, 30)] + ["y"] * 5000
    iv = bnp.Interval(names, np.arange(len(names)), np.arange(len(names)) * 10 ** 10)
    assert _text(iv) == wo.dump_lines(wo.bed_columns(names, np.arange(len(names)), np.arange(len(names)) * 10 ** 10))


@pytest.mark.parametrize("slice_bytes", [1, 7, 4099])
def test_writer_slices_give_the_same_file(tmp_path, monkeypatch, slice_bytes):
    entries, want = _bed6(np.random.default_rng(4), 2000)
    monkeypatch.setattr(bw, "SLICE_BYTES", slice_bytes)
    path = str(tmp_path / "x.bed")
    with bnp.open(path, "w", buffer_type=bnp.io.Bed6Buffer) as f:
        f.write(entries)
    assert open(path, "rb").read() == want


def test_gzip_append_and_streams(tmp_path):
    rng = np.random.default_rng(5)
    parts = [_bed6(rng, n, names=("chr1", "chr2")) for n in (100, 1, 3000)]
    gz = str(tmp_path / "x.bed.gz")
    with pytest.raises(NotImplementedError, match="buffer_type"):
        bnp.open(gz, "w")                                             # BED is written with its buffer type named
    with bnp.open(gz, "w", buffer_type=bnp.io.BedBuffer) as f:
        f.write(parts[0][0])
    with bnp.open(gz, "a", buffer_type=bnp.io.Bed6Buffer) as f:
        f.write(p[0] for p in parts[1:])
    assert gzip.open(gz).read() == b"".join(p[1] for p in parts)
    # a BED file read in chunks and written back: its first three columns
    src = os.path.join(GOLDEN, "ctcf.bed.gz")
    out = str(tmp_path / "ctcf.bed")
    with bnp.open(out, "w", buffer_type=bnp.io.BedBuffer) as f:
        f.write(bnp.open(src).read_chunks(min_chunk_size=100_000))
    text = gzip.open(src).read()
    assert open(out, "rb").read() == b"".join(b"\t".join(l.split(b"\t")[:3]) + b"\n" for l in text.splitlines())
    # Bed6 read with '.' scores writes them as 0
    bed6 = bnp.open(os.path.join(GOLDEN, "alignments.bed"), buffer_type=bnp.io.Bed6Buffer).read()
    cols = io_.parse_delimited(open(os.path.join(GOLDEN, "alignments.bed"), "rb").read(), io_.BED6)[1]
    assert _text(bed6) == wo.dump_lines(list(zip(("text", "int", "int", "text", "int", "strand"), cols)))
    small = os.path.join(GOLDEN, "small_interval.bed")
    assert _text(bnp.open(small).read()) == open(small, "rb").read()


def test_fastq_writes_through_the_buffer_protocol(tmp_path):
    entries = bnp.SequenceEntryWithQuality(["r1", "r2"], ["ACGT", "GG"], ["IIII", "!!"])
    path = str(tmp_path / "x.fq")
    with bnp.open(path, "w") as f:
        f.write(entries)
    assert open(path, "rb").read() == b"@r1\nACGT\n+\nIIII\n@r2\nGG\n+\n!!\n"


def test_ten_million_lines():
    n = 10_000_000
    text, ci, start, stop = io_.synthetic_bed(n, ["chr1", "chr2", "chrX", "chr10"], seed=6)
    names = ["chr1", "chr2", "chrX", "chr10"]
    table = np.frombuffer(b"".join(x.encode() for x in names), dtype=np.uint8)
    offs = np.cumsum([0] + [len(x) for x in names])[:-1]
    dev = "cuda"
    chrom = bnp.EncodedRaggedArray(bnp.EncodedArray(torch.from_numpy(table.copy()).to(dev), bnp.BaseEncoding),
                                   torch.from_numpy(np.array([len(x) for x in names], np.int32)[ci]).to(dev),
                                   starts=torch.from_numpy(offs[ci].astype(np.int64)).to(dev))
    iv = bnp.Interval(chrom, torch.from_numpy(start).to(dev), torch.from_numpy(stop).to(dev))
    assert _text(iv) == text
