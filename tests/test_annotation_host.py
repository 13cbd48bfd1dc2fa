"""GTF/GFF annotations without a GPU: the annotation oracle against the reference's own expectations for its example
files, its attribute rules at their edges, and the C entry point's argument checks."""
import ctypes
import os

import pytest

from bionumpy_b200 import _native as nv

import annotation_oracle as ao

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _path(name):
    return os.path.join(GOLDEN, name)


def test_small_gtf():
    """tests/test_gtf.py: 2 transcripts, 3 exons, the first transcript's gene_id, and the sequences on 'A' * 40000."""
    rows = ao.read(_path("small.gtf"), False)
    tx = ao.select(rows, "transcript", False)
    exons = ao.select(rows, "exon", False)
    assert len(tx) == 2 and len(exons) == 3
    assert tx[0]["gene_id"] == b"ENST00000619216.1"
    seqs = ao.transcript_sequences(exons, lambda c, s, e: (b"A" * 40000)[s:e])
    assert [s for _, s in seqs] == [b"T" * (rows[0]["stop"] - rows[0]["start"]), b"A" * 588]


def test_small_gff():
    """tests/test_gtf.py test_read_gff, and the feature counts of small_gff.gff3 (its ##sequence-region lines inside
    the file are dropped)."""
    rows = ao.read(_path("small_gff.gff3.gz"), True)
    genes = ao.select(rows, "gene", True)
    assert genes[0]["gene_id"] == b"ENSG00000290825.1"
    assert (len(genes), len(ao.select(rows, "transcript", True)), len(ao.select(rows, "exon", True))) == (9, 13, 39)


def test_saccer_gtf():
    rows = ao.read(_path("sacCer3.ensGene.gtf.gz"), False)
    assert len(ao.select(rows, "transcript", False)) == 7127
    assert len(ao.select(rows, "exon", False)) == 7507


def test_gencode_order_agrees_with_the_reference_where_it_should():
    """The reference joins exons in file order; sorting by start agrees on every '+' and every single-exon transcript,
    and GENCODE's '-' transcripts of several exons are the ones it differs on."""
    rows = ao.read(_path("gencode_chr21_head.gtf.gz"), False)
    exons = ao.select(rows, "exon", False)
    def fetch(c, s, e):
        return bytes(b"ACGT"[(i * 7 + i // 3) % 4] for i in range(s, e))

    ours = ao.transcript_sequences(exons, fetch)
    theirs = ao.reference_order_sequences(exons, fetch)
    groups = ao.transcripts(exons)
    assert len(ours) == len(theirs) == len(groups)
    differ = 0
    for (tid, strand, group), a, b in zip(groups, ours, theirs):
        if strand != 1 or len(group) == 1:
            assert a == b, tid
        else:
            differ += a != b
    assert differ == 114


@pytest.mark.parametrize("text, keys, gff, want", [
    (b'gene_id "g1"; transcript_id "t1";', ["gene_id", "transcript_id"], False, {"gene_id": b"g1", "transcript_id": b"t1"}),
    (b'havana_gene_id "h"; gene_idx "x"; gene_id "g"', ["gene_id"], False, {"gene_id": b"g"}),
    (b'gene_id "a;b"; gene_id "c";', ["gene_id"], False, {"gene_id": b"a;b"}),
    (b'gene_id ""; level 2 ;', ["gene_id", "level"], False, {"gene_id": b"", "level": b"2"}),
    (b'  gene_id   plain value  ;x "y"', ["gene_id", "x"], False, {"gene_id": b"plain value", "x": b"y"}),
    (b'gene_id "open;', ["gene_id"], False, {"gene_id": b"open;"}),
    (b'gene_id;gene_id ;', ["gene_id"], False, {"gene_id": b""}),
    (b"ID=a;Parent=b,c;gene_id=g%3B", ["Parent", "gene_id"], True, {"Parent": b"b,c", "gene_id": b"g%3B"}),
    (b"gene_id=x=y; gene_id=z", ["gene_id"], True, {"gene_id": b"x=y"}),
    (b"gene_idx=1;Xgene_id=2", ["gene_id"], True, {}),
])
def test_attribute_rules(text, keys, gff, want):
    got = ao.attribute_values(text, keys, gff)
    assert {k: text[s:s + n] for k, (s, n) in got.items()} == want


def test_missing_attribute_and_comment_lines():
    data = (b"##gff-version 3\nc\ts\tgene\t1\t5\t.\t+\t.\tID=a;gene_id=g1\n###\n"
            b"##sequence-region c 1 9\nc\ts\tgene\t2\t6\t.\t-\t.\tID=b\n")
    rows = ao.read(data, True)
    assert [r["line"] for r in rows] == [0, 3]
    with pytest.raises(ao.Fault) as e:
        ao.select(rows, "gene", True)
    assert e.value.line == 1 and e.value.what == "gene_id"
    with pytest.raises(ao.Fault) as e:
        ao.parse(b"c\ts\tgene\t1\t5\t.\t+\t.\tx\n#\nc\ts\tgene\t1\t5\t.\t*\t.\tx\n", True)
    assert e.value.line == 2


def test_transcript_sequences_case_and_bad_bytes():
    exons = [{"chromosome": b"c", "start": s, "stop": e, "strand": st, "transcript_id": t}
             for s, e, st, t in ((4, 6, 1, b"t1"), (0, 2, 1, b"t1"), (2, 4, 0, b"t2"))]
    seq = b"acGTnA"
    assert ao.transcript_sequences(exons, lambda c, s, e: seq[s:e]) == [(b"t1", b"TNGT"), (b"t2", b"GT")]
    with pytest.raises(ao.BadBase) as e:
        ao.transcript_sequences(exons, lambda c, s, e: b"acGTxA"[s:e])
    assert e.value.offset == 1          # t1 is "-": its last exon, "xA", comes first as "Tx"


def test_attribute_values_argument_checks():
    """BNPK_E_BADARG for 0 or 9 keys, an empty key and an unknown mode, before any device work (no GPU needed)."""
    lib = nv.load_library()
    keys = ctypes.create_string_buffer(b"gene_id" * 9)

    def call(n_keys, offsets, mode=nv.ATTR_GTF):
        offs = (ctypes.c_int64 * len(offsets))(*offsets)
        return lib.bnpk_attribute_values(None, 0, None, None, 0, None, ctypes.cast(keys, ctypes.c_void_p),
                                         ctypes.cast(offs, ctypes.c_void_p), n_keys, mode, None, None, None, None)

    assert call(0, [0]) == nv.E_BADARG
    assert call(9, [7 * i for i in range(10)]) == nv.E_BADARG
    assert call(1, [0, 0]) == nv.E_BADARG
    assert call(1, [0, 33]) == nv.E_BADARG
    assert call(1, [0, 7], mode=2) == nv.E_BADARG
    assert call(8, [7 * i for i in range(9)]) == 0          # no rows: nothing to do


def test_suffixes():
    from bionumpy_b200.io.files import _buffer_type_for
    from bionumpy_b200.io.delimited import GFFBuffer, GTFBuffer
    assert _buffer_type_for(".gtf") is GTFBuffer
    assert _buffer_type_for(".gff") is GFFBuffer and _buffer_type_for(".gff3") is GFFBuffer
    with pytest.raises(RuntimeError, match="does not have a default buffer type"):
        _buffer_type_for(".vcf")


def test_writing_is_refused(tmp_path):
    import bionumpy_b200 as bnp
    for name in ("x.gtf", "x.gff3.gz"):
        with pytest.raises(NotImplementedError):
            bnp.open(str(tmp_path / name), "w")
    assert not os.listdir(tmp_path)
