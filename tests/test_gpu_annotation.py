"""GTF/GFF reading, attribute values, feature selection, annotations on a genome and spliced transcript sequences on
the GPU (bnpk_attribute_values in csrc/interval_kernels.cu, io/delimited.py, datatypes.py, sequence/genes.py) against
the plain-Python restatement in tests/annotation_oracle.py, field for field and byte for byte."""
import gzip
import os
import random
import shutil

import numpy as np
import pytest
import torch

import bionumpy_b200 as bnp
from bionumpy_b200 import _native as nv
from bionumpy_b200 import ops
from bionumpy_b200.io import FormatException, GFFBuffer, GTFBuffer
from bionumpy_b200.rows import RowView
from bionumpy_b200.sequence import get_transcript_sequences

import annotation_oracle as ao

gpu = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
FILES = [("small.gtf", False), ("small_gff.gff3.gz", True), ("sacCer3.ensGene.gtf.gz", False),
         ("gencode_chr21_head.gtf.gz", False)]
POISON = b'\t"; gene_id "p";=\n'


def _path(name):
    return os.path.join(GOLDEN, name)


def _texts(field):
    """The rows of a text field as bytes, with three device-to-host copies."""
    rows = RowView(field)
    base, starts, lens = rows.base.cpu().numpy().tobytes(), rows.starts.cpu().tolist(), rows.lens.cpu().tolist()
    return [base[s:s + n] for s, n in zip(starts, lens)]


def _assert_record(got, want, extra=()):
    assert len(got) == len(want)
    for f in ao.FIELDS + tuple(extra):
        value = getattr(got, f)
        if f in ("start", "stop"):
            assert value.cpu().tolist() == [r[f] for r in want], f
        elif f == "strand":
            assert value.raw().cpu().tolist() == [r[f] for r in want], f
        else:
            assert _texts(value) == [r[f] for r in want], f


def _view(text, off):
    buf = torch.frombuffer(bytearray(b"x" * off + text + POISON * 4), dtype=torch.uint8).cuda()
    return buf[off:off + len(text)]


def _check_features(entries, rows, gff):
    for feature, method in (("gene", "get_genes"), ("transcript", "get_transcripts"), ("exon", "get_exons")):
        try:
            want = ao.select(rows, feature, gff)
        except ao.Fault as e:
            with pytest.raises(FormatException) as got:
                getattr(entries, method)()
            assert got.value.line_number == e.line and e.what in str(got.value)
            continue
        _assert_record(getattr(entries, method)(), want, ao.KEYS[feature])


@gpu
@pytest.mark.parametrize("name, gff", FILES)
def test_whole_files(name, gff):
    entries = bnp.open(_path(name)).read()
    assert isinstance(entries, bnp.GFFEntry if gff else bnp.GTFEntry)
    rows = ao.read(_path(name), gff)
    _assert_record(entries, rows)
    _check_features(entries, rows, gff)


@gpu
@pytest.mark.parametrize("name, gff", FILES)
@pytest.mark.parametrize("chunk_size", [700, 5000, 100000])
def test_chunks(name, gff, chunk_size, tmp_path):
    """read_chunks at several sizes, from the file and from its .gz form: the chunks' rows joined are the file's."""
    raw = ao.read_file(_path(name))
    plain = tmp_path / name.replace(".gz", "")
    plain.write_bytes(raw)
    gz = tmp_path / (plain.name + ".gz")
    gz.write_bytes(gzip.compress(raw))
    rows = ao.read(raw, gff)
    for path in (str(plain), str(gz)):
        got = []
        for chunk in bnp.open(path).read_chunks(min_chunk_size=chunk_size):
            got += list(zip(_texts(chunk.chromosome), chunk.start.cpu().tolist(), _texts(chunk.atributes)))
        assert got == [(r["chromosome"], r["start"], r["atributes"]) for r in rows]


@gpu
@pytest.mark.parametrize("off", range(16))
def test_chunk_placement(off):
    for name, gff in FILES[:2]:
        text = ao.split_header(ao.read_file(_path(name)))
        buf = (GFFBuffer if gff else GTFBuffer).from_raw_buffer(_view(text, off))
        rows, _ = ao.parse(text, gff)
        entries = buf.get_data()
        _assert_record(entries, rows)
        _check_features(entries, rows, gff)


def _random_attributes(rng, gff, keys):
    """One attribute column and the keys it holds, drawn from prefixes/suffixes of the keys, duplicates, quotes with
    ';' inside, unquoted and empty values, spaces and long padding."""
    parts = []
    for _ in range(rng.choice([0, 1, 2, 3, 5, 8, 20, 60])):
        k = rng.choice(keys + [k + "x" for k in keys] + ["x" + k for k in keys] + [k[:-1] for k in keys] +
                       ["tag", "level", "a"])
        v = rng.choice(["", "v", "ab;cd", "  sp ace  ", "x" * rng.randrange(1, 400), "q\"q", "=", "1,2"])
        if gff:
            parts.append(f"{' ' * rng.randrange(2)}{k}={v.replace(';', ',')}")
        elif rng.random() < 0.7:
            parts.append(f"{' ' * rng.randrange(2)}{k}{' ' * rng.randrange(1, 3)}\"{v.replace(chr(34), '')}\"")
        else:
            parts.append(f"{' ' * rng.randrange(2)}{k} {v.replace(';', '').replace(chr(34), '')}")
    text = ";".join(parts) + (";" if rng.random() < 0.5 else "") + (" " if rng.random() < 0.2 else "")
    return text.encode()


@gpu
@pytest.mark.parametrize("gff", [False, True])
@pytest.mark.parametrize("seed", range(4))
def test_random_attribute_columns(gff, seed):
    """The kernel alone on random rows of 0 to > 2000 bytes, every key and a row mask, against the oracle."""
    rng = random.Random(seed)
    keys = ["gene_id", "transcript_id", "exon_id", "gene_name", "id"][: rng.randrange(1, 6)]
    rows = [_random_attributes(rng, gff, keys) for _ in range(3000)]
    rows[0] = (";".join(f"{k}={'y' * 700}" if gff else f'{k} "{"y" * 700}"' for k in keys * 3)).encode()
    select = [rng.random() < 0.8 for _ in rows]
    text = b"".join(rows)
    assert max(map(len, rows)) > 2000 or seed
    starts = np.cumsum([0] + [len(r) for r in rows[:-1]])
    base = _view(text, seed)
    st = torch.tensor(starts, dtype=torch.int64, device="cuda")
    ln = torch.tensor([len(r) for r in rows], dtype=torch.int32, device="cuda")
    sel = torch.tensor(select, dtype=torch.uint8, device="cuda")
    v_starts, v_lens, status = ops.attribute_values(base, st, ln, keys, nv.ATTR_GFF if gff else nv.ATTR_GTF, sel)
    v_starts, v_lens = v_starts.cpu().tolist(), v_lens.cpu().tolist()
    first_missing = None
    for r, (row, s) in enumerate(zip(rows, select)):
        if not s:
            assert all(v_lens[k][r] == 0 and v_starts[k][r] == starts[r] for k in range(len(keys)))
            continue
        got = ao.attribute_values(row, keys, gff)
        for k, key in enumerate(keys):
            if key in got:
                assert (v_starts[k][r] - starts[r], v_lens[k][r]) == got[key], (r, key, row)
            elif first_missing is None:
                first_missing = (r, k)
    fault = ops.read_status(status).column_fault()
    assert (None if fault is None else fault[:2]) == first_missing
    if fault is not None:
        assert fault[2] == nv.BAD_ATTRIBUTE


GTF_LINE = 'c\ts\t{f}\t{a}\t{b}\t.\t{st}\t.\t{attr}'


@gpu
@pytest.mark.parametrize("where", ["first", "middle", "last"])
@pytest.mark.parametrize("crlf", [False, True])
def test_missing_attribute_row(where, crlf):
    lines = [GTF_LINE.format(f="exon", a=i, b=i + 5, st="+", attr=f'gene_id "g{i}"; transcript_id "t{i}"; '
                             f'exon_id "e{i}";') for i in range(50)]
    bad = {"first": 0, "middle": 23, "last": 49}[where]
    lines[bad] = lines[bad].replace('exon_id "e', 'exon_idx "e')
    lines.insert(10, GTF_LINE.format(f="gene", a=1, b=2, st="-", attr='gene_id "g"'))
    text = ("\r\n" if crlf else "\n").join(lines).encode() + (b"\r\n" if crlf else b"\n")
    entries = GTFBuffer.from_raw_buffer(_view(text, 3)).get_data()
    with pytest.raises(FormatException) as e:
        entries.get_exons()
    assert e.value.line_number == bad + (bad >= 10) and "exon_id" in str(e.value)
    assert _texts(entries.get_genes().gene_id) == [b"g"]
    assert len(entries.get_transcripts()) == 0


@gpu
def test_gff_internal_comments_and_fault_lines():
    text = (b"c\ts\tgene\t1\t5\t.\t+\t.\tID=a;gene_id=g1\n###\n##sequence-region c 1 9\n"
            b"c\ts\tgene\t2\t6\t.\t-\t.\tgene_id=g2;x=1\n#c\n")
    entries = GFFBuffer.from_raw_buffer(_view(text, 5)).get_data()
    assert _texts(entries.get_genes().gene_id) == [b"g1", b"g2"]
    with pytest.raises(FormatException) as e:
        GFFBuffer.from_raw_buffer(_view(text + b"c\ts\tgene\t2\t6\t.\t*\t.\tx\n", 0))
    assert e.value.line_number == 5


def _sacCer3_fasta(tmp_path):
    fa = tmp_path / "sacCer3.fa"
    with gzip.open(_path("sacCer3.fa.gz")) as src, open(fa, "wb") as dst:
        shutil.copyfileobj(src, dst)
    return str(fa)


def _fasta_dict(path):
    seqs, name = {}, None
    for line in open(path, "rb"):
        line = line.rstrip(b"\r\n")
        if line.startswith(b">"):
            name = line[1:].split()[0]
            seqs[name] = []
        else:
            seqs[name].append(line)
    return {k: b"".join(v) for k, v in seqs.items()}


@gpu
def test_annotation_on_a_genome(tmp_path):
    """Genome.read_annotation: exon, transcript and intron masks against a dense oracle, and the interval classes."""
    fa = _sacCer3_fasta(tmp_path)
    genome = bnp.Genome.from_file(fa)
    ann = genome.read_annotation(_path("sacCer3.ensGene.gtf.gz"))
    exons, tx = ann.exons, ann.transcripts
    assert isinstance(exons, bnp.genomic_data.Exons) and isinstance(exons[exons.start.cpu() > 0], bnp.genomic_data.Exons)
    assert len(tx) == 7127 and len(exons) == 7507
    rows = ao.read(_path("sacCer3.ensGene.gtf.gz"), False)
    sizes = genome.get_chromosome_sizes()
    dense = {}
    for feature in ("exon", "transcript"):
        m = {c: np.zeros(n, dtype=bool) for c, n in sizes.items()}
        for r in ao.select(rows, feature, False):
            if r["chromosome"].decode() in m:
                m[r["chromosome"].decode()][r["start"]:r["stop"]] = True
        dense[feature] = m
    introns = tx.get_mask() & ~exons.get_mask()
    for c in sizes:
        assert np.array_equal(np.asarray(exons.get_mask()[c]), dense["exon"][c]), c
        assert np.array_equal(np.asarray(introns[c]), dense["transcript"][c] & ~dense["exon"][c]), c
    assert _texts(exons.transcript_id) == [r["transcript_id"] for r in ao.select(rows, "exon", False)
                                           if r["chromosome"].decode() in sizes]
    assert len(exons.merged()) <= len(exons) and len(exons.sorted()) == len(exons)


@gpu
def test_transcript_sequences_sacCer3(tmp_path):
    fa = _sacCer3_fasta(tmp_path)
    entries = bnp.open(_path("sacCer3.ensGene.gtf.gz")).read()
    genome = _fasta_dict(fa)
    exons = ao.select(ao.read(_path("sacCer3.ensGene.gtf.gz"), False), "exon", False)
    want = ao.transcript_sequences(exons, lambda c, s, e: genome[c][s:e])
    got = get_transcript_sequences(entries, bnp.open_indexed(fa))
    assert len(want) == 7127
    assert _texts(got.name) == [t for t, _ in want] and _texts(got.sequence) == [s for _, s in want]
    out = tmp_path / "transcripts.fa"
    with bnp.open(str(out), "w") as f:
        f.write(got)
    assert out.stat().st_size > sum(len(s) for _, s in want)
    one = genome[b"chrI"]
    chr1 = [e for e in exons if e["chromosome"] == b"chrI"]
    on_chr1 = np.array([i for i, c in enumerate(_texts(entries.chromosome)) if c == b"chrI"])
    got = get_transcript_sequences(entries[on_chr1], bnp.as_encoded_array(one.decode()))
    assert _texts(got.sequence) == [s for _, s in ao.transcript_sequences(chr1, lambda c, s, e: one[s:e])]


@gpu
def test_transcript_sequences_small_gtf():
    entries = bnp.open(_path("small.gtf")).read()
    got = get_transcript_sequences(entries, bnp.as_encoded_array("A" * 40000))
    assert _texts(got.sequence) == [b"T" * 67, b"A" * 588]
    assert len(get_transcript_sequences(entries[np.zeros(0, dtype=np.int64)], "ACGT")) == 0


@gpu
def test_transcript_sequences_gencode_head(tmp_path):
    """The GENCODE head on a seeded random chr21/chr22 with lower-case stretches, then with one bad byte."""
    rng = np.random.default_rng(7)
    sizes = {"chr21": 46709983, "chr22": 50818468}
    genome = {}
    for c, n in sizes.items():
        seq = np.frombuffer(b"ACGT", dtype=np.uint8)[rng.integers(0, 4, n)].copy()
        for s in rng.integers(0, n - 10000, 200):
            seq[s:s + 5000] += 32
        genome[c] = seq
    rows = ao.read(_path("gencode_chr21_head.gtf.gz"), False)
    exons = ao.select(rows, "exon", False)
    bad_at = exons[40]["start"] + 3
    genome["chr21"][bad_at] = ord("x")

    def write(path):
        """60 bases a line, and its .fai"""
        with open(path, "wb") as f, open(str(path) + ".fai", "w") as fai:
            for c, seq in genome.items():
                f.write(b">" + c.encode() + b"\n")
                fai.write(f"{c}\t{len(seq)}\t{f.tell()}\t60\t61\n")
                n_full = len(seq) // 60
                lines = np.concatenate([seq[:n_full * 60].reshape(-1, 60), np.full((n_full, 1), 10, dtype=np.uint8)], 1)
                f.write(lines.tobytes())
                if len(seq) % 60:
                    f.write(seq[n_full * 60:].tobytes() + b"\n")

    fa = tmp_path / "g.fa"
    write(fa)
    entries = bnp.open(_path("gencode_chr21_head.gtf.gz")).read()
    fetch = lambda c, s, e: genome[c.decode()][s:e].tobytes()
    with pytest.raises(ao.BadBase) as want:
        ao.transcript_sequences(exons, fetch)
    with pytest.raises(bnp.EncodingError) as got:
        get_transcript_sequences(entries, bnp.open_indexed(str(fa)))
    assert got.value.offset == want.value.offset
    genome["chr21"][bad_at] = ord("a")
    write(fa)
    want = ao.transcript_sequences(exons, fetch)
    got = get_transcript_sequences(entries, bnp.open_indexed(str(fa)))
    assert _texts(got.name) == [t for t, _ in want] and _texts(got.sequence) == [s for _, s in want]


@gpu
def test_attribute_values_argument_checks():
    lib = nv.load_library()
    base = torch.zeros(8, dtype=torch.uint8, device="cuda")
    st = torch.zeros(2, dtype=torch.int64, device="cuda")
    ln = torch.zeros(2, dtype=torch.int32, device="cuda")
    before = lib.bnpk_launch_count()
    with pytest.raises(nv.NativeLibraryError):
        ops.attribute_values(base.cpu(), st, ln, ["gene_id"])
    with pytest.raises(TypeError):
        ops.attribute_values(base, st.to(torch.int32), ln, ["gene_id"])
    with pytest.raises(ValueError):
        ops.attribute_values(base, st, ln, ["k"] * 9)
    with pytest.raises(TypeError):
        ops.attribute_values(base, st, ln, ["gene_id"], select=torch.ones(2, dtype=torch.int32, device="cuda"))
    assert lib.bnpk_launch_count() == before
    from bionumpy_b200 import torch_ops
    top = torch_ops.load()
    starts, lens, status = top.attribute_values(base, st, ln, ["gene_id"], nv.ATTR_GTF, None)
    assert starts.shape == (1, 2) and lens.cpu().tolist() == [[0, 0]]
    assert ops.read_status(status).column_fault() == (0, 0, nv.BAD_ATTRIBUTE)
