"""SAM on the GPU against tests/sam_oracle.py: every field of the five SAM fixtures read whole, in chunks, at a cut on
every line border and from .sam.gz (gzip and BGZF); the four SAM/BAM twin pairs and a SAM twin of the CTCF BAM down to
their pileups; chunk views at every byte offset with poison after them; random lines (11 columns, many tags, empty
text columns, lines of more than 512 bytes and of 200 kB, CRLF, '*' fields); malformed lines and integers; CIGARs of
0 to 3000 ops and invalid CIGARs; and the argument checks of the three K16 ops and their dispatcher ops."""
import gzip
import os

import numpy as np
import pytest
import torch

import bam_oracle as bo
import pileup_oracle as po
import sam_oracle as so
import bionumpy_b200 as bnp
from bionumpy_b200 import _native as nv
from bionumpy_b200 import ops, torch_ops
from bionumpy_b200.io.bam import BamIntervalBuffer
from bionumpy_b200.io.exceptions import FormatException
from bionumpy_b200.io.sam import SAMBuffer, SAMIntervalBuffer

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
TWINS = ["alignments", "many_alignments", "small_alignments", "test"]
FIXTURES = ["sam_spec_example"] + TWINS
CTCF = "ctcf_chr21-22_every6th"
TEXT = ("name", "chromosome", "cigar", "next_chromosome", "sequence", "quality", "extra")
GOOD = b"r\t0\tc\t1\t0\t*\t*\t0\t0\t*\t*"


def _golden(name):
    with open(os.path.join(GOLDEN, name), "rb") as f:
        return f.read()


def _texts(x):
    data = x.ravel().raw().cpu().numpy().tobytes()
    ends = np.cumsum(x.lengths.cpu().numpy().astype(np.int64))
    return [data[a:b] for a, b in zip(np.concatenate([[0], ends[:-1]]), ends)]


def _rows(x):
    flat = x.ravel()
    flat = (flat.raw() if hasattr(flat, "raw") else flat).cpu().numpy().astype(np.int64)
    ends = np.cumsum(x.lengths.cpu().numpy().astype(np.int64))
    return [flat[a:b].tolist() for a, b in zip(np.concatenate([[0], ends[:-1]]), ends)]


def check_entries(e, recs):
    """Every field of the SAMEntry chunk e equals the oracle's records."""
    assert type(e) is bnp.SAMEntry and len(e) == len(recs)
    for f in so.FIELDS:
        v = getattr(e, f)
        if f in TEXT:
            assert _texts(v) == [r[f] for r in recs], f
        else:
            assert v.dtype == torch.int64 and v.is_cuda
            assert v.cpu().tolist() == [r[f] for r in recs], f


def check_bed6(b, rows):
    assert len(b) == len(rows)
    assert [t.decode() for t in _texts(b.chromosome)] == [r[0] for r in rows]
    assert b.start.cpu().tolist() == [r[1] for r in rows]
    assert b.stop.cpu().tolist() == [r[2] for r in rows]
    assert [t.decode() for t in _texts(b.name)] == [r[3] for r in rows]
    assert b.score.cpu().tolist() == [r[4] for r in rows]
    assert ["+-"[c] for c in b.strand.raw().cpu().tolist()] == [r[5] for r in rows]


def _write(tmp_path, data, name="x.sam"):
    p = str(tmp_path / name)
    with open(p, "wb") as f:
        f.write(data)
    return p


def _entries(chunks):
    """The records of the chunks of a reader, field by field, as oracle dicts."""
    out = []
    for e in chunks:
        cols = {f: (_texts(getattr(e, f)) if f in TEXT else getattr(e, f).cpu().tolist()) for f in so.FIELDS}
        out += [dict(zip(so.FIELDS, vals)) for vals in zip(*[cols[f] for f in so.FIELDS])]
    return out


@pytest.mark.parametrize("name", FIXTURES)
def test_fixture_whole_chunked_and_gzipped(name, tmp_path):
    data = _golden(name + ".sam")
    recs, fault = so.read_sam(data)
    assert fault is None
    p = os.path.join(GOLDEN, name + ".sam")
    check_entries(bnp.open(p).read(), recs)
    assert bnp.count_entries(p) == len(recs)
    for size in ((1, 97, 4096) if len(data) < 5000 else (97, 4096)):
        with bnp.open(p) as f:
            assert _entries(f.read_chunks(min_chunk_size=size)) == recs
    gz = _write(tmp_path, gzip.compress(data), "x.sam.gz")
    bg = _write(tmp_path, bo.bgzf(data, block=1000), "y.sam.gz")
    for q in (gz, bg):
        check_entries(bnp.open(q).read(), recs)
        with bnp.open(q) as f:
            assert _entries(f.read_chunks(min_chunk_size=500)) == recs


@pytest.mark.parametrize("name", FIXTURES)
def test_cut_at_every_line_border(name):
    """from_raw_buffer of the record lines cut 1 to 5 bytes past each line border keeps exactly the lines before it."""
    _, lines = so.split_lines(_golden(name + ".sam"))
    recs, _ = so.read_lines(lines)
    body = b"".join(x + b"\n" for x in lines)
    border = 0
    for k, line in enumerate(lines):
        border += len(line) + 1
        for extra in (1, 5):
            buf = SAMBuffer.from_raw_buffer(body[:border + extra])
            assert buf.size == border and buf.n_lines == k + 1
            check_entries(buf.get_data(), recs[:k + 1])


@pytest.mark.parametrize("name", TWINS)
def test_sam_and_bam_twins_agree(name):
    s = bnp.open(os.path.join(GOLDEN, name + ".sam")).read()
    b = bnp.open(os.path.join(GOLDEN, name + ".bam")).read()
    assert len(s) == len(b) > 0
    assert _texts(s.name) == _texts(b.name) and _texts(s.chromosome) == _texts(b.chromosome)
    assert s.flag.cpu().tolist() == b.flag.cpu().tolist() and s.mapq.cpu().tolist() == b.mapq.cpu().tolist()
    assert (s.position - 1).cpu().tolist() == b.position.cpu().tolist()
    op, length = bnp.alignments.parse_cigar(s.cigar)
    assert op.encoding == bnp.encodings.CigarOpEncoding and length.ravel().dtype == torch.int64
    assert _rows(op) == _rows(b.cigar_op) and _rows(length) == _rows(b.cigar_length)
    seq = [t if t != b"*" else b"" for t in _texts(s.sequence)]
    assert seq == [bo.seq_text(r).encode() for r in _rows(b.sequence)]
    qual = [[c - 33 for c in t] if t != b"*" else [] for t in _texts(s.quality)]
    assert qual == _rows(b.quality)
    check_same_bed6(bnp.alignments.alignment_to_interval(s), bnp.alignments.alignment_to_interval(b))
    si = bnp.open(os.path.join(GOLDEN, name + ".sam"), buffer_type=SAMIntervalBuffer).read()
    bi = bnp.open(os.path.join(GOLDEN, name + ".bam"), buffer_type=BamIntervalBuffer).read()
    check_same_bed6(si, bi)


def check_same_bed6(a, b):
    assert len(a) == len(b)
    for f in ("chromosome", "name"):
        assert _texts(getattr(a, f)) == _texts(getattr(b, f)), f
    for f in ("start", "stop", "score"):
        assert getattr(a, f).cpu().tolist() == getattr(b, f).cpu().tolist(), f
    assert a.strand.raw().cpu().tolist() == b.strand.raw().cpu().tolist()


def test_ctcf_sam_twin_gives_the_bam_pileup(tmp_path):
    names, _, recs, _ = bo.read_bam(os.path.join(GOLDEN, CTCF + ".bam"))
    header = b"".join(b"@SQ\tSN:%s\tLN:1\n" % n.encode() for n in names)
    text = so.bam_to_sam(names, recs, header)
    p = _write(tmp_path, text)
    g = bnp.Genome.from_file(os.path.join(GOLDEN, "chr21-22.chrom.sizes"))
    from_sam = g.read_intervals(p).get_pileup()
    from_bam = g.read_intervals(os.path.join(GOLDEN, CTCF + ".bam")).get_pileup()
    sizes = dict((a, int(b)) for a, b in (line.split() for line in open(os.path.join(GOLDEN, "chr21-22.chrom.sizes"))))
    rows = so.bed6_rows(so.read_sam(text)[0], placed_only=True)
    check_bed6(bnp.open(p, buffer_type=SAMIntervalBuffer).read(), rows)
    for name, size in sizes.items():
        s, e, v = po.runs_of(po.dense_pileup([r[1] for r in rows if r[0] == name], [r[2] for r in rows if r[0] == name],
                                             size))
        for got in (from_sam[name], from_bam[name]):
            assert got.starts.cpu().tolist() == s.tolist() and got.ends.cpu().tolist() == e.tolist()
            assert got.values.cpu().tolist() == v.tolist()


def test_chunk_views_at_every_offset_with_poison_after():
    _, lines = so.split_lines(_golden("sam_spec_example.sam"))
    body = b"".join(x + b"\n" for x in lines)
    recs, _ = so.read_lines(lines)
    poison = b"\t9\t\t*\t" * 8
    for off in range(16):
        raw = b"\t" * off + body + poison
        big = torch.from_numpy(np.frombuffer(raw, dtype=np.uint8).copy()).cuda()
        view = big[off:off + len(body)]
        buf = SAMBuffer.from_raw_buffer(view)
        assert buf.size == len(body)
        check_entries(buf.get_data(), recs)
        b = SAMIntervalBuffer.from_raw_buffer(view).get_data()
        check_bed6(b, so.bed6_rows(recs, placed_only=True))


def _random_line(rng, long_bytes=0):
    def text(lo, hi, alphabet=b"ACGTN"):
        return bytes(rng.choice(np.frombuffer(alphabet, dtype=np.uint8), int(rng.integers(lo, hi))))
    n = int(rng.integers(0, 300)) if not long_bytes else long_bytes
    seq = text(n, n + 1) if rng.random() > 0.1 else b"*"
    qual = bytes(rng.integers(33, 75, len(seq)).astype(np.uint8)) if seq != b"*" and rng.random() > 0.1 else b"*"
    ops_ = [(int(rng.integers(0, 9)), int(rng.integers(0, 1000))) for _ in range(int(rng.integers(0, 6)))]
    cols = [text(0, 30, b"abcdefXYZ0123456789_.:"),
            str(int(rng.integers(0, 4096))).encode(),
            b"*" if rng.random() < 0.1 else text(0, 8, b"chr12XYM"),
            str(int(rng.integers(-5, 1 << 30))).encode(), b"+" + str(int(rng.integers(0, 256))).encode(),
            so.cigar_text(ops_).encode(), rng.choice([b"*", b"=", b"chr2", b""]),
            str(int(rng.integers(0, 1 << 30))).encode(), str(int(rng.integers(-1000, 1000))).encode(), seq, qual]
    n_tags = int(rng.choice([0, 0, 1, 3, 40]))
    tags = [b"X%d:i:%d" % (t, int(rng.integers(0, 1000))) for t in range(n_tags)]
    return b"\t".join(cols + tags)


@pytest.mark.parametrize("crlf", [False, True])
def test_random_lines(tmp_path, crlf):
    rng = np.random.default_rng(11 + crlf)
    lines = [_random_line(rng) for _ in range(3000)]
    lines += [_random_line(rng, 700), _random_line(rng, 2000), _random_line(rng, 200_000), GOOD, GOOD + b"\t"]
    rng.shuffle(lines)
    end = b"\r\n" if crlf else b"\n"
    data = b"@HD\tVN:1.6" + end + b"".join(x + end for x in lines)
    recs, fault = so.read_sam(data)
    assert fault is None and len(recs) == len(lines)
    assert any(len(x) > 512 for x in lines) and any(r["extra"] == b"" for r in recs)
    p = _write(tmp_path, data)
    e = bnp.open(p).read()
    check_entries(e, recs)
    with bnp.open(p) as f:
        assert _entries(f.read_chunks(min_chunk_size=50_000)) == recs
    check_bed6(bnp.alignments.alignment_to_interval(e), so.bed6_rows(recs))
    check_bed6(bnp.open(p, buffer_type=SAMIntervalBuffer).read(), so.bed6_rows(recs, placed_only=True))
    op, length = bnp.alignments.parse_cigar(e.cigar)
    want = [so.parse_cigar(r["cigar"]) for r in recs]
    assert _rows(op) == [[o for o, _ in w] for w in want] and _rows(length) == [[n for _, n in w] for w in want]


def _malformed(at, n=300, line=None):
    lines = [GOOD.replace(b"r\t", b"r%d\t" % i, 1) for i in range(n)]
    if line is not None:
        lines[at] = line
    return b"".join(x + b"\n" for x in lines)


@pytest.mark.parametrize("at", [0, 150, 299])
def test_ten_columns_name_their_line_across_chunks(tmp_path, at):
    data = _malformed(at, line=b"\t".join(GOOD.split(b"\t")[:10]))
    assert so.read_sam(data)[1] == (at, 10, so.BAD_COLUMNS)
    p = _write(tmp_path, data)
    for size in (None, 700, 2000):
        with pytest.raises(FormatException) as err:
            with bnp.open(p) as f:
                f.read() if size is None else list(f.read_chunks(min_chunk_size=size))
        assert err.value.line_number == at


@pytest.mark.parametrize("col", [1, 3, 4, 7, 8])
@pytest.mark.parametrize("bad", [b"12a", b"", b"-", b"1" * 19])
def test_bad_integer_names_its_line(tmp_path, col, bad):
    cols = GOOD.split(b"\t")
    cols[col] = bad
    at = 123
    data = _malformed(at, line=b"\t".join(cols))
    assert so.read_sam(data)[1] == (at, col, so.BAD_INT)
    p = _write(tmp_path, data)
    for size in (None, 1000):
        with pytest.raises(FormatException) as err:
            with bnp.open(p) as f:
                f.read() if size is None else list(f.read_chunks(min_chunk_size=size))
        assert err.value.line_number == at


def test_first_fault_wins():
    lines = [GOOD] * 10
    lines[7] = b"\t".join(GOOD.split(b"\t")[:4])
    cols = GOOD.split(b"\t")
    cols[8] = b"x"
    lines[4] = b"\t".join(cols)
    data = b"".join(x + b"\n" for x in lines)
    assert so.read_sam(data)[1] == (4, 8, so.BAD_INT)
    with pytest.raises(FormatException) as err:
        SAMBuffer.from_raw_buffer(data)
    assert err.value.line_number == 4


def test_random_cigars_up_to_3000_ops():
    rng = np.random.default_rng(5)
    want = [[(int(rng.integers(0, 9)), int(rng.integers(0, 10 ** int(rng.integers(1, 10)))))
             for _ in range(int(n))] for n in np.concatenate([rng.integers(0, 12, 500), [0, 1, 3000, 2999]])]
    texts = [so.cigar_text(w) for w in want]
    op, length = bnp.alignments.parse_cigar(texts)
    assert _rows(op) == [[o for o, _ in w] for w in want] and _rows(length) == [[n for _, n in w] for w in want]
    ref = bnp.alignments.count_reference_length(op, length).cpu().tolist()
    assert ref == [so.reference_length(w) for w in want]


@pytest.mark.parametrize("cigar", [b"", b"M", b"10", b"10M5", b"10Q", b"1234567890M"])
def test_invalid_cigar_raises_where_it_is_parsed(tmp_path, cigar):
    lines = [GOOD.replace(b"\t*\t*\t0", b"\t5M\t*\t0", 1)] * 20
    cols = lines[0].split(b"\t")
    cols[5] = cigar
    lines[13] = b"\t".join(cols)
    data = b"".join(x + b"\n" for x in lines)
    recs, fault = so.read_sam(data)
    assert fault is None and so.first_bad_cigar(recs) == 13
    p = _write(tmp_path, data)
    e = bnp.open(p).read()                      # a file with an invalid CIGAR still reads as SAMEntry
    check_entries(e, recs)
    for call in (lambda: bnp.alignments.parse_cigar(e.cigar), lambda: bnp.alignments.alignment_to_interval(e),
                 lambda: bnp.open(p, buffer_type=SAMIntervalBuffer).read()):
        with pytest.raises(FormatException) as err:
            call()
        assert err.value.line_number == 13


def test_selection_and_reference_snippet():
    reads = bnp.open(os.path.join(GOLDEN, "sam_spec_example.sam")).read()
    recs, _ = so.read_sam(_golden("sam_spec_example.sam"))
    primary = reads[(reads.flag & 0x904) == 0]
    keep = [r for r in recs if r["flag"] & 0x904 == 0]
    check_entries(primary, keep)
    op, length = bnp.alignments.parse_cigar(primary.cigar)
    clipped = primary[op[..., 0] == "S"]
    assert _texts(clipped.name) == [r["name"] for r in keep if so.parse_cigar(r["cigar"])[0][0] == 4]
    assert _texts(reads.extra)[-1] == b"NM:i:1"


# ---- argument checks --------------------------------------------------------------------------------------------
def _u8(data):
    return torch.from_numpy(np.frombuffer(data, dtype=np.uint8).copy()).cuda()


def _args():
    chunk = _u8(b"".join(x + b"\n" for x in (GOOD, GOOD)))
    starts, lens, _ = ops.line_split(chunk, 1, 0, 0, ord("@"), False, 0, max_rows=2)
    base = _u8(b"5M*3S2M")
    c_starts = torch.tensor([0, 2, 3], dtype=torch.int64, device="cuda")
    c_lens = torch.tensor([2, 1, 4], dtype=torch.int32, device="cuda")
    offsets = torch.tensor([0, 1, 1, 3], dtype=torch.int64, device="cuda")
    return dict(chunk=chunk, starts=starts, lens=lens, base=base, c_starts=c_starts, c_lens=c_lens, offsets=offsets,
                status=nv.new_status("cuda"))


CALLS = {
    "sam_columns": lambda a: ops.sam_columns(a["chunk"], a["starts"], a["lens"], a["status"]),
    "cigar_count": lambda a: ops.cigar_count(a["base"], a["c_starts"], a["c_lens"], a["status"]),
    "cigar_unpack": lambda a: ops.cigar_unpack(a["base"], a["c_starts"], a["c_lens"], a["offsets"], 3),
}
DISPATCH = {
    "sam_columns": lambda a: torch_ops.load().sam_columns(a["chunk"], a["starts"], a["lens"]),
    "cigar_count": lambda a: torch_ops.load().cigar_count(a["base"], a["c_starts"], a["c_lens"]),
    "cigar_unpack": lambda a: torch_ops.load().cigar_unpack(a["base"], a["c_starts"], a["c_lens"], a["offsets"], 3),
}
BAD = {"sam_columns": [("chunk", lambda t: t.cpu()), ("chunk", lambda t: torch.stack([t, t], 1)[:, 0]),
                       ("starts", lambda t: t[:-1]), ("lens", lambda t: t.long()), ("status", lambda t: t[:4])],
       "cigar_count": [("base", lambda t: t.cpu()), ("c_starts", lambda t: t.int()), ("c_lens", lambda t: t[:-1]),
                       ("status", lambda t: t.cpu())],
       "cigar_unpack": [("base", lambda t: t.long()), ("c_starts", lambda t: t[:-1]), ("offsets", lambda t: t[:-1]),
                        ("offsets", lambda t: t.cpu())]}


def test_valid_arguments_give_the_same_values_both_ways():
    a = _args()
    fields, _ = ops.sam_columns(a["chunk"], a["starts"], a["lens"])
    assert torch.equal(fields, DISPATCH["sam_columns"](a)[0])
    assert fields[nv.SAM_F_POS].cpu().tolist() == [1, 1]
    counts, ref_len, _ = ops.cigar_count(a["base"], a["c_starts"], a["c_lens"])
    d_counts, d_ref, _ = DISPATCH["cigar_count"](a)
    assert counts.cpu().tolist() == d_counts.cpu().tolist() == [1, 0, 2]
    assert ref_len.cpu().tolist() == d_ref.cpu().tolist() == [5, 0, 2]
    op, length = ops.cigar_unpack(a["base"], a["c_starts"], a["c_lens"], a["offsets"], 3)
    d_op, d_length = DISPATCH["cigar_unpack"](a)
    assert op.cpu().tolist() == d_op.cpu().tolist() == [0, 4, 0]
    assert length.cpu().tolist() == d_length.cpu().tolist() == [5, 3, 2]


class _NoLibrary:
    def __getattr__(self, name):
        def called(*args):
            pytest.fail(f"a rejected argument reached {name}")
        return called


@pytest.mark.parametrize("case", [(op, i) for op in BAD for i in range(len(BAD[op]))])
def test_rejected_argument_launches_nothing(case, monkeypatch):
    op, i = case
    name, bad = BAD[op][i]
    for calls in (CALLS, DISPATCH) if name != "status" else (CALLS,):
        a = _args()
        a[name] = bad(a[name])
        torch_ops.load()
        torch.cuda.synchronize()
        before = nv.load_library().bnpk_launch_count()
        with monkeypatch.context() as m:
            m.setattr(ops, "lib", lambda: _NoLibrary())
            with pytest.raises((TypeError, ValueError, RuntimeError)):
                calls[op](a)
        assert nv.load_library().bnpk_launch_count() == before
