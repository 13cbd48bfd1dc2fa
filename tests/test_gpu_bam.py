"""BAM on the GPU against tests/bam_oracle.py: every field of every record of the five fixtures and of synthetic files
(every base code and cigar op, empty and odd sequences, no cigar, missing qualities, refID -1, a header of 100 k
contigs, a 200 kb record, a record border at every offset of a segment), decoy records that make the speculative
split guess wrong, chunk cuts at and next to every record border, malformed records, and what is built on the
records: intervals, reference lengths, selection, counts, FASTQ and read pileups."""
import os

import numpy as np
import pytest
import torch

import bam_oracle as bo
import pileup_oracle as po
import bionumpy_b200 as bnp
from bionumpy_b200 import _native as nv
from bionumpy_b200 import ops
from bionumpy_b200.io.bam import BamIntervalBuffer
from bionumpy_b200.io.exceptions import FormatException

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
# the header and every sixth record of the reference's ctcf_chr21-22.bam (coordinate-sorted, chr21 and chr22)
CTCF = "ctcf_chr21-22_every6th"
FIXTURES = ["alignments", "many_alignments", "small_alignments", "test", CTCF]
NAMES = [f"chr{i}" for i in range(5)]


def _path(name):
    return os.path.join(GOLDEN, name + ".bam")


def _texts(x):
    data = x.ravel().raw().cpu().numpy().tobytes()
    ends = np.cumsum(x.lengths.cpu().numpy().astype(np.int64))
    return [data[a:b] for a, b in zip(np.concatenate([[0], ends[:-1]]), ends)]


def _rows(x):
    flat = x.ravel()
    flat = flat.raw() if hasattr(flat, "raw") else flat
    flat = flat.cpu().numpy().astype(np.int64)
    ends = np.cumsum(x.lengths.cpu().numpy().astype(np.int64))
    return [flat[a:b].tolist() for a, b in zip(np.concatenate([[0], ends[:-1]]), ends)]


def check_entries(e, names, recs):
    """Every field of the BamEntry chunk e equals the oracle's records."""
    assert len(e) == len(recs)
    assert [t.decode() for t in _texts(e.chromosome)] == [bo.chromosome(r, names) for r in recs]
    assert _texts(e.name) == [r["name"] for r in recs]
    for field, key in (("flag", "flag"), ("position", "pos"), ("mapq", "mapq")):
        v = getattr(e, field)
        assert v.dtype == torch.int64 and v.is_cuda
        assert v.cpu().tolist() == [r[key] for r in recs], field
    assert e.cigar_op.encoding == bnp.encodings.CigarOpEncoding
    assert _rows(e.cigar_op) == [[op for op, _ in r["cigar"]] for r in recs]
    assert e.cigar_length.ravel().dtype == torch.int64
    assert _rows(e.cigar_length) == [[n for _, n in r["cigar"]] for r in recs]
    assert e.sequence.encoding == bnp.encodings.BamEncoding
    assert _rows(e.sequence) == [r["seq"] for r in recs]
    assert e.quality.ravel().dtype == torch.uint8
    assert _rows(e.quality) == [list(r["qual"]) for r in recs]


def check_bed6(b, rows):
    assert [t.decode() for t in _texts(b.chromosome)] == [r[0] for r in rows]
    assert b.start.cpu().tolist() == [r[1] for r in rows]
    assert b.stop.cpu().tolist() == [r[2] for r in rows]
    assert [t.decode() for t in _texts(b.name)] == [r[3] for r in rows]
    assert b.score.cpu().tolist() == [r[4] for r in rows]
    assert ["+-"[c] for c in b.strand.raw().cpu().tolist()] == [r[5] for r in rows]


@pytest.mark.parametrize("name", FIXTURES)
def test_fixture_every_field(name):
    names, _, recs, _ = bo.read_bam(_path(name))
    e = bnp.open(_path(name)).read()
    check_entries(e, names, recs)
    b = bnp.open(_path(name), buffer_type=bnp.io.bam.BamIntervalBuffer).read()
    check_bed6(b, bo.bed6_rows(recs, names, placed_only=True))
    assert bnp.count_entries(_path(name)) == len(recs)


def test_reference_bam_tests():
    e = bnp.open(_path("small_alignments")).read()
    assert e[:4].position.cpu().tolist() == [523205, 3837782, 907877, 260353]
    assert [t.decode() for t in _texts(e[:4].chromosome)] == ["contig28", "contig14", "contig23", "contig11"]
    assert e[e.mapq == 60].position[:4].cpu().tolist() == [523205, 3837782, 907877, 406696]
    assert bnp.open(_path("test"), buffer_type=BamIntervalBuffer).read().start[0].item() == 7512371


def _synthetic(tmp_path, recs, names=NAMES, text=b"", block=65280, name="x.bam"):
    p = str(tmp_path / name)
    bo.write_bam(p, names, [1 << 30] * len(names), recs, text, block)
    return p


def test_synthetic_every_case(tmp_path):
    rng = np.random.default_rng(1)
    recs = bo.random_records(rng, 2000, len(NAMES), unmapped=0.1)
    recs += [dict(ref_id=-1, pos=-1, name=b"*", seq=[], qual=b"", cigar=[]),                     # unmapped, l_seq 0
             dict(ref_id=2, pos=5, name=b"odd", seq=list(range(16)) + [3], qual=None,            # 0xFF quality
                  cigar=[(op, op + 1) for op in range(9)]),
             dict(ref_id=1, pos=7, name=b"nocigar", seq=[1, 2, 4], qual=b"\x00\x01\x02", cigar=[], flag=4)]
    p = _synthetic(tmp_path, recs, block=7000)
    names, _, want, _ = bo.read_bam(p)
    e = bnp.open(p).read()
    check_entries(e, names, want)
    check_bed6(bnp.open(p, buffer_type=BamIntervalBuffer).read(), bo.bed6_rows(want, names, placed_only=True))
    check_bed6(bnp.alignments.alignment_to_interval(e), bo.bed6_rows(want, names))
    assert bnp.alignments.count_reference_length(e.cigar_op, e.cigar_length).cpu().tolist() == \
        [bo.reference_length(r["cigar"]) for r in want]
    counts = bnp.count_encoded(e.sequence.ravel(), axis=None).counts.cpu().numpy()
    assert counts.tolist() == np.bincount(np.concatenate([r["seq"] for r in want]).astype(np.int64),
                                          minlength=16).tolist()
    sel = e[(e.flag & 16) != 0]
    assert sel.position.cpu().tolist() == [r["pos"] for r in want if r["flag"] & 16]
    assert _texts(sel.name) == [r["name"] for r in want if r["flag"] & 16]
    assert bnp.count_entries(p) == len(want)
    with bnp.open(p, buffer_type=BamIntervalBuffer) as f:
        assert sum(len(c) for c in f.read_chunks(min_chunk_size=5000)) == sum(r["ref_id"] >= 0 for r in want)


def test_large_header_and_long_record(tmp_path):
    names = [f"contig_{i}" for i in range(100_000)]
    text = b"@CO\t" + b"x" * (3 << 20) + b"\n"
    rng = np.random.default_rng(2)
    recs = bo.random_records(rng, 50, len(names))
    recs.insert(20, dict(ref_id=99_999, pos=3, name=b"long", seq=[int(x) for x in rng.integers(0, 16, 200_001)],
                         cigar=[(0, 200_001)]))
    p = _synthetic(tmp_path, recs, names, text)
    names, _, want, _ = bo.read_bam(p)
    for chunk in (None, 1 << 20, 70_000):
        with bnp.open(p) as f:
            parts = [f.read()] if chunk is None else list(f.read_chunks(min_chunk_size=chunk))
        k = 0
        for part in parts:
            check_entries(part, names, want[k:k + len(part)])
            k += len(part)
        assert k == len(want)


def test_record_border_at_every_segment_offset():
    """Records of 37 + i bytes, i = 0, 1, 2, ...: record starts fall at every offset of a segment of every size."""
    recs = [bo.record_bytes(ref_id=0, name=b"", l_name=1, seq=[], aux=bytes(i % 200)) for i in range(3000)]
    data = b"".join(recs)
    want = np.cumsum([0] + [len(r) for r in recs[:-1]]).tolist()
    d = torch.frombuffer(bytearray(data), dtype=torch.uint8).cuda()
    for seg in (64, 100, 257, 1024, 4096, 8192):
        starts, status = ops.bam_split(d, 1, seg)
        st = ops.read_status(status)
        assert st.n_records == len(recs) and st.n_complete_bytes == len(data)
        assert st.words[nv.ST_BAD_BASE] == nv.INT64_MAX
        assert starts[:len(recs)].cpu().tolist() == want
        ends = np.array(want) + np.array([len(r) for r in recs])
        for cut in (len(data) - 1, want[-1], want[-1] + 1, want[1500] + 3):
            starts, status = ops.bam_split(d[:cut].clone(), 1, seg)
            st = ops.read_status(status)
            k = int((ends <= cut).sum())
            assert st.n_records == k and st.n_complete_bytes == int(ends[k - 1])
            assert starts[:k].cpu().tolist() == want[:k]


def _decoy_chain():
    return b"".join(bo.record_bytes(ref_id=0, name=b"d", seq=[1, 2, 3], qual=b"\x05\x06\x07") for _ in range(3))


def test_decoys_make_speculation_walk_again_and_the_split_stays_exact(tmp_path):
    chain = _decoy_chain()
    rng = np.random.default_rng(3)
    recs = []
    for i in range(40):
        recs += bo.random_records(rng, 5, len(NAMES))
        payload = chain * int(rng.integers(200, 2000))
        aux = b"ZBBC" + len(payload).to_bytes(4, "little") + payload
        recs.append(dict(ref_id=1, pos=i, name=b"decoy%d" % i, seq=[1] * 10, cigar=[(0, 10)], aux=aux))
    p = _synthetic(tmp_path, recs)
    names, _, want, offsets = bo.read_bam(p)
    e = bnp.open(p).read()
    check_entries(e, names, want)
    data = bo.gzip.decompress(open(p, "rb").read())
    body = torch.frombuffer(bytearray(data[offsets[0]:]), dtype=torch.uint8).cuda()
    for seg in (256, 1024, 4096, 16384):
        starts, status = ops.bam_split(body, len(NAMES), seg)
        st = ops.read_status(status)
        assert st.n_values > 0, seg
        assert st.n_records == len(want)
        assert starts[:len(want)].cpu().tolist() == [o - offsets[0] for o in offsets]


def test_ctcf_speculation_never_walks_again():
    names, _, recs, offsets = bo.read_bam(_path(CTCF))
    data = bo.gzip.decompress(open(_path(CTCF), "rb").read())
    body = torch.frombuffer(bytearray(data[offsets[0]:]), dtype=torch.uint8).cuda()
    starts, status = ops.bam_split(body, len(names))
    st = ops.read_status(status)
    assert st.n_values == 0 and st.n_records == len(recs)
    assert starts[:len(recs)].cpu().tolist() == [o - offsets[0] for o in offsets]


def test_chunk_cuts_at_every_record_border(tmp_path):
    rng = np.random.default_rng(4)
    recs = bo.random_records(rng, 150, len(NAMES), read_len=(0, 40), aux_len=(0, 10))
    p = _synthetic(tmp_path, recs, block=500)
    names, _, want, _ = bo.read_bam(p)
    whole = bnp.open(p).read()
    check_entries(whole, names, want)
    for m in list(range(1, 90, 3)) + [333, 1000, 4097]:
        k = 0
        with bnp.open(p) as f:
            for part in f.read_chunks(min_chunk_size=m):
                check_entries(part, names, want[k:k + len(part)])
                k += len(part)
        assert k == len(want), m


MALFORMED = {
    "block_size": (dict(block_size=20), nv.BAM_BAD_BLOCK_SIZE),
    "l_read_name": (dict(l_name=0), nv.BAM_BAD_NAME),
    "cigar_op": (dict(cigar=[(0, 5), (9, 5)]), nv.BAM_BAD_CIGAR_OP),
    "ref_id": (dict(ref_id=len(NAMES)), nv.BAM_BAD_REF_ID),
    "next_ref_id": (dict(next_ref_id=-2), nv.BAM_BAD_REF_ID),
    "sizes": (dict(l_seq=1000), nv.BAM_BAD_SIZES),
}


@pytest.mark.parametrize("case", list(MALFORMED))
@pytest.mark.parametrize("at", [0, 37, 400])
def test_malformed_record_names_its_record(tmp_path, case, at):
    rng = np.random.default_rng(6)
    good = [bo.record_bytes(**r) for r in bo.random_records(rng, 500, len(NAMES))]
    kw, kind = MALFORMED[case]
    bad = bo.record_bytes(**{**dict(ref_id=0, name=b"bad", seq=[1, 2, 3]), **kw})
    p = _synthetic(tmp_path, good[:at] + [bad] + good[at:], block=3000)
    for chunk in (None, 997, 20_000):
        with pytest.raises(FormatException) as exc:
            with bnp.open(p) as f:
                if chunk is None:
                    f.read()
                else:
                    for _ in f.read_chunks(min_chunk_size=chunk):
                        pass
        assert exc.value.line_number == at, (chunk, str(exc.value))
        assert bnp.io.bam.FAULTS[kind] in str(exc.value)


@pytest.mark.parametrize("cut", [1, 4, 30, 36, 50])
def test_truncated_last_record(tmp_path, cut):
    rng = np.random.default_rng(7)
    recs = [bo.record_bytes(**r) for r in bo.random_records(rng, 60, len(NAMES), read_len=(40, 80))]
    data = bo.header_bytes(NAMES, [100] * len(NAMES)) + b"".join(recs)
    p = str(tmp_path / "t.bam")
    open(p, "wb").write(bo.bgzf(data[:len(data) - len(recs[-1]) + cut]))
    for chunk in (None, 500):
        with pytest.raises(FormatException, match="ends inside a record") as exc:
            with bnp.open(p) as f:
                f.read() if chunk is None else list(f.read_chunks(min_chunk_size=chunk))
        assert exc.value.line_number == 59


def test_fault_at_a_segment_start():
    """A bad record that starts exactly at a segment border, found by speculation and by the resolve pass alike."""
    seg = 1024
    recs = [bo.record_bytes(ref_id=0, name=b"", l_name=1, seq=[], aux=bytes(seg - 37)) for _ in range(5)]
    bad = bo.record_bytes(ref_id=0, name=b"", l_name=1, seq=[], block_size=8)
    d = torch.frombuffer(bytearray(b"".join(recs) + bad + b"".join(recs)), dtype=torch.uint8).cuda()
    for s in (seg, seg // 2, 4096):
        _, status = ops.bam_split(d, 1, s)
        st = ops.read_status(status)
        assert st.n_records == 5 and st.n_complete_bytes == 5 * seg
        assert st.words[nv.ST_BAD_BASE] == 5 << 8 | nv.BAM_BAD_BLOCK_SIZE


def test_bam_to_fastq_is_byte_equal(tmp_path):
    rng = np.random.default_rng(8)
    recs = bo.random_records(rng, 500, len(NAMES))
    for r in recs:
        r["qual"] = bytes(q % 90 for q in r["qual"])
    p = _synthetic(tmp_path, recs)
    _, _, want, _ = bo.read_bam(p)
    e = bnp.open(p).read()
    out = str(tmp_path / "x.fq")
    with bnp.open(out, "w") as f:
        f.write(bnp.SequenceEntryWithQuality(e.name, e.sequence, e.quality))
    assert open(out, "rb").read() == bo.fastq_text(want)
    assert bnp.open(_path("small_alignments")).read().cigar_op[..., 0].raw().cpu().tolist() == \
        [r["cigar"][0][0] for r in bo.read_bam(_path("small_alignments"))[2]]


def test_ctcf_read_pileup_on_chr21_22():
    sizes = dict((a, int(b)) for a, b in (line.split() for line in open(os.path.join(GOLDEN, "chr21-22.chrom.sizes"))))
    g = bnp.Genome.from_file(os.path.join(GOLDEN, "chr21-22.chrom.sizes"))
    pileup = g.read_intervals(_path(CTCF)).get_pileup()
    names, _, recs, _ = bo.read_bam(_path(CTCF))
    rows = bo.bed6_rows(recs, names, placed_only=True)
    for name, size in sizes.items():
        starts = [r[1] for r in rows if r[0] == name]
        stops = [r[2] for r in rows if r[0] == name]
        s, e, v = po.runs_of(po.dense_pileup(starts, stops, size))
        got = pileup[name]
        assert got.starts.cpu().tolist() == s.tolist() and got.ends.cpu().tolist() == e.tolist()
        assert got.values.cpu().tolist() == v.tolist()
