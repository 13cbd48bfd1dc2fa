"""BAM without a GPU: the oracle against the reference's own BAM test values and the SAM twins of the fixtures, the
serialiser against the parser, the package's host header parser against the oracle, and writing .bam still refused."""
import os
import struct

import numpy as np
import pytest

import bam_oracle as bo
from bionumpy_b200.io import bam as pkg_bam
from bionumpy_b200.io.exceptions import FormatException

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
TWINS = ["alignments", "many_alignments", "small_alignments", "test"]


def _path(name):
    return os.path.join(GOLDEN, name)


def test_oracle_reproduces_the_reference_bam_tests():
    """tests/test_bam.py of the reference: small_alignments.bam read as BamEntry, selected by mapq, and test.bam as
    intervals."""
    names, _, recs, _ = bo.read_bam(_path("small_alignments.bam"))
    assert [r["pos"] for r in recs[:4]] == [523205, 3837782, 907877, 260353]
    assert [bo.chromosome(r, names) for r in recs[:4]] == ["contig28", "contig14", "contig23", "contig11"]
    assert [bo.seq_text(r["seq"]) for r in recs[:2]] == [
        "CNATCTCTTTCGTACGAGTATTTCGCGTTCTTGAGGTGAGCCTGTTAAGATCCAAATCGTTAAATAGCCGATTTCGGCTCTCGCAGTAAATTTTATAGCCATCACCTTTTCA"
        "TCAATCAGCTCGCACGGCTCTACGAACCTTCGAGTTCAC",
        "TTTGGCGTTAGCCACGTTTCTGACGTATAAAATGAAGCCGAGAAATCGAATCGCTGATTGCTTCATGCATCTATCATATGCCGCTGAAGAACGAGGGATCGTATGCAGCTT"
        "TTACTTTCTCAAGAACGAACGTCGGCTATTGGCTGTTTTA"]
    assert [r["name"] for r in recs[:2]] == [b"ERR6054981.1", b"ERR6054981.1"]
    assert [r["pos"] for r in recs if r["mapq"] == 60][:4] == [523205, 3837782, 907877, 406696]
    names, _, recs, _ = bo.read_bam(_path("test.bam"))
    assert bo.bed6_rows(recs, names, placed_only=True)[0][1] == 7512371


@pytest.mark.parametrize("name", TWINS)
def test_oracle_agrees_with_the_sam_twin(name):
    names, _, recs, _ = bo.read_bam(_path(name + ".bam"))
    sam = bo.parse_sam(_path(name + ".sam"))
    assert len(recs) == len(sam) > 0
    for r, s in zip(recs, sam):
        assert r["name"] == s["name"] and r["flag"] == s["flag"] and r["pos"] == s["pos"] and r["mapq"] == s["mapq"]
        assert bo.chromosome(r, names) == s["chromosome"]
        assert bo.cigar_text(r["cigar"]) == s["cigar"]
        assert bo.seq_text(r["seq"]) == s["seq"]
        assert r["qual"] == s["qual"]


def test_ctcf_fixture_is_sorted_on_chr21_and_chr22():
    """ctcf_chr21-22_every6th.bam: the header and every sixth record of the reference's ctcf_chr21-22.bam."""
    names, lengths, recs, _ = bo.read_bam(_path("ctcf_chr21-22_every6th.bam"))
    assert len(recs) == 10295
    sizes = dict(line.split() for line in open(_path("chr21-22.chrom.sizes")))
    assert {bo.chromosome(r, names) for r in recs} <= set(sizes)
    keys = [(r["ref_id"], r["pos"]) for r in recs]
    assert keys == sorted(keys)


def test_serialiser_and_parser_round_trip():
    rng = np.random.default_rng(5)
    names = [f"c{i}" for i in range(7)]
    recs = bo.random_records(rng, 300, len(names), unmapped=0.2)
    recs.append(dict(ref_id=-1, pos=-1, name=b"*", seq=[], qual=b"", cigar=[]))
    data = bo.header_bytes(names, [100] * 7, b"@HD\tVN:1.6\n") + b"".join(bo.record_bytes(**r) for r in recs)
    got_names, got_lengths, got, _ = bo.parse_bam(data)
    assert got_names == names and got_lengths == [100] * 7
    for r, g in zip(recs, got):
        for k, v in r.items():
            assert g[k] == (bytes(v) if k == "qual" else v), k
    assert bo.parse_bam(bo.gzip.decompress(bo.bgzf(data, block=1000)))[2] == got


@pytest.mark.parametrize("name", TWINS + ["ctcf_chr21-22_every6th"])
def test_host_header_parser_agrees_with_the_oracle(name):
    data = bo.gzip.decompress(open(_path(name + ".bam"), "rb").read())
    names, lengths, size = bo.parse_header(data)
    h = pkg_bam.parse_header(data)
    assert (h.names, h.lengths, h.size) == (names, lengths, size)
    assert h.info == list(zip(names, lengths))
    for cut in (0, 3, 8, size // 2, size - 1):         # a header cut short is incomplete, not an error
        assert pkg_bam.parse_header(data[:cut]) is None


def test_host_header_parser_large_header_and_errors():
    names = [f"contig_{i}" for i in range(100_000)]
    text = b"@CO\t" + b"x" * 3_000_000 + b"\n"
    data = bo.header_bytes(names, list(range(100_000)), text)
    h = pkg_bam.parse_header(data)
    assert h.names == names and h.lengths == list(range(100_000)) and h.size == len(data)
    with pytest.raises(FormatException):
        pkg_bam.parse_header(b"BAX\1" + bytes(20))
    with pytest.raises(FormatException):
        pkg_bam.parse_header(b"BAM\1" + struct.pack("<i", -1) + bytes(8))


def test_writing_bam_still_raises(tmp_path):
    import bionumpy_b200 as bnp
    for mode in ("w", "a"):
        with pytest.raises(RuntimeError, match="does not have a default buffer type"):
            bnp.open(str(tmp_path / "x.bam"), mode)


def test_not_gzip_raises(tmp_path):
    import bionumpy_b200 as bnp
    p = tmp_path / "x.bam"
    p.write_bytes(b"BAM\1" + bytes(100))
    with pytest.raises(FormatException, match="not gzip"):
        bnp.open(str(p))
