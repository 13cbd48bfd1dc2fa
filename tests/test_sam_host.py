"""SAM without a GPU: the oracle against the reference's SAM expectations and against the BAM oracle's decoding of the
four BAM twins, the CIGAR grammar, the header mirror, the K16 kernels' machine code, and writing .sam still refused."""
import os
import re
import shutil
import subprocess

import pytest

import bam_oracle as bo
import sam_oracle as so
from bionumpy_b200 import _native as nv

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TWINS = ["alignments", "many_alignments", "small_alignments", "test"]


def _read(name):
    with open(os.path.join(GOLDEN, name), "rb") as f:
        return f.read()


def test_oracle_reads_the_sam_spec_example():
    """io_tests/test_sam.py of the reference: the spec example reads as 8 records and extra[-1] is NM:i:1; the
    CT:Z: tag, with its ';' and space, stays whole in extra."""
    header, lines = so.split_lines(_read("sam_spec_example.sam"))
    assert len(header) == 2
    recs, fault = so.read_lines(lines)
    assert fault is None and len(recs) == 8
    assert recs[-1]["extra"] == b"NM:i:1"
    assert recs[2]["name"] == b"*" and recs[2]["extra"] == b"CT:Z:.;Warning;Note=Ref wrong?"
    assert recs[2]["sequence"] == b"*" and recs[2]["quality"] == b"*"
    assert recs[0]["extra"] == b"" and recs[5]["extra"] == b""
    assert [r["position"] for r in recs] == [1, 7, 8, 9, 9, 18, 31, 39]
    assert recs[7]["length"] == -41 and recs[7]["next_chromosome"] == b"="
    assert so.bed6_rows(recs)[1] == ("ref", 6, 24, "r001", 30, "+")


def test_oracle_reads_the_two_alignments_with_pos_as_written():
    recs, fault = so.read_sam(_read("alignments.sam"))
    assert fault is None and len(recs) == 2
    assert [r["position"] for r in recs] == [1706, 1706]
    assert [r["cigar"] for r in recs] == [b"25M", b"24M"]
    assert recs[0]["extra"].split(b"\t")[0] == b"AS:i:0" and recs[0]["extra"].endswith(b"YT:Z:UU")


@pytest.mark.parametrize("name", TWINS)
def test_oracle_agrees_with_the_bam_twin(name):
    names, _, bam, _ = bo.read_bam(os.path.join(GOLDEN, name + ".bam"))
    sam, fault = so.read_sam(_read(name + ".sam"))
    assert fault is None and len(sam) == len(bam) > 0
    for s, b in zip(sam, bam):
        assert s["name"] == b["name"] and s["flag"] == b["flag"] and s["mapq"] == b["mapq"]
        assert s["chromosome"].decode() == bo.chromosome(b, names)
        assert s["position"] - 1 == b["pos"]
        assert so.parse_cigar(s["cigar"]) == [tuple(x) for x in b["cigar"]]
        assert (s["sequence"] if s["sequence"] != b"*" else b"") == bo.seq_text(b["seq"]).encode()
        assert (bytes(q - 33 for q in s["quality"]) if s["quality"] != b"*" else b"") == b["qual"]
    assert so.bed6_rows(sam, placed_only=True) == bo.bed6_rows(bam, names, placed_only=True)


def test_bam_to_sam_round_trips_through_the_oracles():
    names, _, bam, _ = bo.read_bam(os.path.join(GOLDEN, "ctcf_chr21-22_every6th.bam"))
    sam, fault = so.read_sam(so.bam_to_sam(names, bam, b"@HD\tVN:1.6"))
    assert fault is None and len(sam) == len(bam)
    assert so.bed6_rows(sam, placed_only=True) == bo.bed6_rows(bam, names, placed_only=True)


@pytest.mark.parametrize("text,ops", [(b"*", []), (b"0M", [(0, 0)]), (b"10M5I3D2N4S1H1P6=7X", [
    (0, 10), (1, 5), (2, 3), (3, 2), (4, 4), (5, 1), (6, 1), (7, 6), (8, 7)]), (b"123456789M", [(0, 123456789)])])
def test_cigar_grammar_accepts(text, ops):
    assert so.parse_cigar(text) == ops


@pytest.mark.parametrize("text", [b"", b"M", b"10", b"10M5", b"10Q", b"1234567890M", b"**", b"*M", b"10m", b" 10M"])
def test_cigar_grammar_refuses(text):
    assert so.parse_cigar(text) is None


def test_oracle_faults():
    good = b"r\t0\tc\t1\t0\t*\t*\t0\t0\t*\t*"
    assert so.read_lines([good, b"\t".join(good.split(b"\t")[:10])])[1] == (1, 10, so.BAD_COLUMNS)
    for col in (1, 3, 4, 7, 8):
        for bad in (b"12a", b"", b"-", b"1" * 19):
            cols = good.split(b"\t")
            cols[col] = bad
            assert so.read_lines([good, good, b"\t".join(cols)])[1] == (2, col, so.BAD_INT)
    assert so.read_lines([good + b"\r", good + b"\r"]) == ([so.read_lines([good])[0][0]] * 2, None)
    assert so.read_lines([b"r\t+5\tc\t-0\t0\t*\t*\t0\t" + b"9" * 18 + b"\t*\t*"])[0][0]["length"] == int("9" * 18)


def test_header_constants_match_the_python_mirror():
    text = open(os.path.join(ROOT, "include", "bnpk.h")).read()
    consts = {m.group(1): int(m.group(2)) for m in re.finditer(r"#define\s+BNPK_(SAM_F_\w+|SAM_FIELDS|BAD_CIGAR)\s+(\d+)",
                                                                text)}
    assert len(consts) == 21
    for name, value in consts.items():
        assert getattr(nv, name) == value, name
    assert nv.BAD_CIGAR == so.BAD_CIGAR and nv.BAD_COLUMNS == so.BAD_COLUMNS and nv.BAD_INT == so.BAD_INT
    for fn in ("bnpk_sam_columns", "bnpk_cigar_count", "bnpk_cigar_unpack"):
        assert fn in nv.SIGNATURES and re.search(rf"\bint {fn}\(", text), fn


def test_sam_kernels_are_sm90a_code_without_stack():
    tool = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(tool):
        pytest.skip("cuobjdump not available")
    out = subprocess.run([tool, "-res-usage", nv.LIB_PATH], capture_output=True, text=True).stdout
    assert "sm_90a" in out
    usage = {m.group(1): (int(m.group(2)), int(m.group(3)))
             for m in re.finditer(r"Function (\S+):\s*REG:(\d+) STACK:(\d+)", out)}
    found = {n: v for n, v in usage.items() if re.search(r"sam_columns_kernel|cigar_count_kernel|cigar_unpack_kernel", n)}
    assert len(found) == 3, sorted(found)
    for name, (regs, stack) in found.items():
        assert stack == 0 and regs <= 64, (name, regs, stack)


def test_suffix_and_writing_still_refused(tmp_path):
    import bionumpy_b200 as bnp
    from bionumpy_b200.io.files import _buffer_type_for
    from bionumpy_b200.io.sam import SAMBuffer
    assert _buffer_type_for(".sam") is SAMBuffer
    assert bnp.io.SAMBuffer is SAMBuffer and bnp.SAMEntry is bnp.datatypes.SAMEntry
    assert bnp.SAMEntry._fields == so.FIELDS
    for name in ("x.sam", "x.sam.gz"):
        for mode in ("w", "a"):
            with pytest.raises(RuntimeError, match="does not have a default buffer type"):
                bnp.open(str(tmp_path / name), mode)
    assert not os.listdir(tmp_path)
    with pytest.raises(NotImplementedError):
        SAMBuffer.from_data(None)
