"""No GPU: the reader oracle (tests/reader_oracle.py) pinned to the reference's goldens, the byte sources of the pinned
reader (plain pread, single-stream gzip, multi-member gzip, BGZF) against file.read(n), and the line split's
dispatcher schema."""
import gzip
import os

import numpy as np
import pytest

import reader_oracle as ro
from bionumpy_b200 import _native as nv
from bionumpy_b200.io import bgzf
from bionumpy_b200.io.ingest import _GzipSource, _PreadSource
from oracle import bnp_oracle as o

FASTQ_TEXT = b"@headerishere\nCTTGTTGA\n+\n!!!!!!!!\n@anotherheader\nCGG\n+\n~~~\n"        # tests/buffers.py
FASTA_TEXT = b">header\nCTTGTTGA\n>header2\nCGG\n"
CR_FASTQ = (b"@test_sequence_id_here\r\nGATTTGGGGTTCAAAGCAGTATCGATCAAATAGTAAATCCATTTGTTCAACTCACAGTTT\r\n+\r\n"
            b"!''*((((***+))%%%++)(%%%%).1***-+*''))**55CCF>>>>>>CCCCCCC65\r\n")            # tests/test_io.py:192-201
CR_FASTA = b">test_sequence_id_here\r\nGACTG\r\n>test_sequence_id_here2\r\nGACTCGAG\r\n"
MALFORMED_FASTQ = [(b"@header\nactg\n-\n!!!!\n", 2), (b"header\nactg\n+\n!!!!\n", 0),            # test_io_exceptions.py
                   (b"@header\nactg\n+\n@header\nactg\n+\n@header\nactg\n+\n", 4)]
VALID_FASTQ = b"@header\nacgtt\n+\n!!!!!\n"


def test_big_fq_chunks_511_then_489(big_fq_bytes):
    for keep in (True, False):
        chunks = ro.read_chunks(big_fq_bytes.tobytes(), 300000, keep_unterminated_last=keep, **ro.FASTQ)
        assert [len(c.records) for c in chunks] == [511, 489]
        assert [c.n_lines_read for c in chunks] == [2044, 4000]
        assert b"".join(c.data for c in chunks) == big_fq_bytes.tobytes()
        size, starts, lens = o.fastq_split(big_fq_bytes)
        raw = big_fq_bytes.tobytes()
        assert chunks[1].records[-1][1] == raw[starts[-1, 1]:starts[-1, 1] + lens[-1, 1]]


def test_buffer_texts():
    assert ro.read_all(FASTQ_TEXT, **ro.FASTQ) == [(b"headerishere", b"CTTGTTGA", b"+", b"!!!!!!!!"),
                                                  (b"anotherheader", b"CGG", b"+", b"~~~")]
    assert ro.read_all(FASTA_TEXT, **ro.FASTA) == [(b"header", b"CTTGTTGA"), (b"header2", b"CGG")]
    for m in range(1, len(FASTQ_TEXT) + 2):
        chunks = ro.read_chunks(FASTQ_TEXT, m, **ro.FASTQ)
        assert [r for c in chunks for r in c.records] == ro.read_all(FASTQ_TEXT, **ro.FASTQ)


def test_carriage_return_fixtures():
    (rec,) = ro.read_all(CR_FASTQ, **ro.FASTQ)
    assert len(rec[1]) == 60 and len(rec[3]) == 60 and rec[0] == b"test_sequence_id_here"
    assert ro.read_all(CR_FASTA, **ro.FASTA) == [(b"test_sequence_id_here", b"GACTG"),
                                                (b"test_sequence_id_here2", b"GACTCGAG")]
    # '\r' on a header of the incomplete tail only: nothing is trimmed (one_line_buffer.py:175-182)
    text = b"@a\nAC\n+\nII\r\n@b\r\nAC"
    (chunk,) = ro.read_chunks(text, 100, keep_unterminated_last=False, **ro.FASTQ)
    assert chunk.records == [(b"a", b"AC", b"+", b"II\r")]


@pytest.mark.parametrize("text,line", MALFORMED_FASTQ)
def test_format_exception_line_numbers(text, line):
    with pytest.raises(ro.ReaderFormatError) as e:
        ro.read_all(text, **ro.FASTQ)
    assert e.value.line_number == line
    with pytest.raises(ro.ReaderFormatError) as e:                          # test_io_exceptions.py:85-100
        ro.read_chunks(VALID_FASTQ * 100 + text, 200, **ro.FASTQ)
    assert e.value.line_number == 4 * 100 + line


def test_two_line_fasta_format_exception():
    with pytest.raises(ro.ReaderFormatError) as e:
        ro.read_all(b">header\nacggtt\nacggtt\n>header\nacgtt\n", **ro.FASTA)
    assert e.value.line_number == 2


def test_unterminated_last_record_deviation():
    text = FASTQ_TEXT[:-1]                                                  # no final newline
    full = ro.read_all(FASTQ_TEXT, **ro.FASTQ)
    for m in range(1, len(text) + 2):
        kept = [r for c in ro.read_chunks(text, m, **ro.FASTQ) for r in c.records]
        ref = [r for c in ro.read_chunks(text, m, keep_unterminated_last=False, **ro.FASTQ) for r in c.records]
        assert kept == full
        assert ref == (full[:1] if len(text) % m == 0 else full)            # the reference loses the last record


def test_truncated_tail_is_never_a_record():
    for cut in (b"@r\nAC\n+\n", b"@r\nAC\n", b"@r\n", b"@r\nAC\n+\nI"):
        text = FASTQ_TEXT + cut
        for m in range(1, len(text) + 2):
            got = [r for c in ro.read_chunks(text, m, **ro.FASTQ) for r in c.records]
            assert got == ro.read_all(FASTQ_TEXT, **ro.FASTQ) + ([(b"r", b"AC", b"+", b"I")] if cut.endswith(b"I") else [])


def test_max_chunk_size_below_one_record():
    with pytest.raises(ro.ReaderNoCompleteEntry):
        ro.read_chunks(FASTQ_TEXT, 4, max_chunk_size=20, **ro.FASTQ)
    assert len(ro.read_chunks(FASTQ_TEXT, 4, max_chunk_size=40, **ro.FASTQ)) == 2


def test_plain_line_split():
    size, starts, lens = ro.plain_line_split(np.frombuffer(b"ab\n\ncd\ne", dtype=np.uint8))
    assert size == 7 and starts.tolist() == [0, 3, 4] and lens.tolist() == [2, 0, 2]


# ---- the byte sources of the pinned reader -----------------------------------------------------------------------
def _text(n_bytes, seed=0):
    rng = np.random.default_rng(seed)
    return bytes(rng.choice(np.frombuffer(b"ACGT\n@+", dtype=np.uint8), size=n_bytes).tolist())


def _drain(src, sizes):
    """Bytes handed out per start/finish with the given read sizes (the last size repeats), and the `last` flags."""
    got, flags, i = [], [], 0
    while True:
        n = sizes[min(i, len(sizes) - 1)]
        buf, nread, last = src.finish(src.start(n))
        got.append(bytes(buf.numpy()[:nread]))
        flags.append(last)
        i += 1
        if last:
            return got, flags


def _write_sources(tmp_path, data):
    plain = tmp_path / "x.fq"
    plain.write_bytes(data)
    gz = tmp_path / "x.fq.gz"
    gz.write_bytes(gzip.compress(data))
    multi = tmp_path / "multi.fq.gz"
    third = len(data) // 3
    multi.write_bytes(b"".join(gzip.compress(data[a:b]) for a, b in ((0, third), (third, 2 * third), (2 * third, len(data)))))
    bg = tmp_path / "bgzf.fq.gz"
    with open(bg, "wb") as f:
        w = bgzf.BgzfWriter(f)
        w.write(data)
        w.close()
    return plain, gz, multi, bg


@pytest.mark.parametrize("kind", ["pread", "gzip", "multi", "bgzf"])
def test_sources_hand_out_file_read_bytes(tmp_path, kind):
    data = _text(3 * bgzf.BLOCK_INPUT + 1234)
    plain, gz, multi, bg = _write_sources(tmp_path, data)
    path = {"pread": plain, "gzip": gz, "multi": multi, "bgzf": bg}[kind]
    B, N = bgzf.BLOCK_INPUT, len(data)
    size_lists = [[B], [B - 1], [B + 1], [N], [N // 2], [1 << 20], [7, B - 7, 2 * B, 1234], [N - 1, 1], [4096]]
    for sizes in size_lists:
        if kind == "pread":
            f = open(path, "rb")
            src = _PreadSource(f)
        else:
            src = _GzipSource(str(path))
            assert src.parallel == (kind == "bgzf")
        got, flags = _drain(src, sizes)
        if kind == "pread":
            f.close()
        with gzip.open(path) if kind != "pread" else open(path, "rb") as ref:
            want, i = [], 0
            while True:
                n = sizes[min(i, len(sizes) - 1)]
                want.append(ref.read(n))
                i += 1
                if len(want[-1]) < n:
                    break
        assert b"".join(got) == data
        # every read but the last hands out exactly what file.read(n) does; the last one is flagged
        assert got[:-1] == want[:len(got) - 1] and flags[-1] and not any(flags[:-1])
        assert b"".join(got[len(got) - 1:]) == b"".join(want[len(got) - 1:])


@pytest.mark.parametrize("kind", ["gzip", "multi", "bgzf"])
def test_last_read_of_zero_bytes(tmp_path, kind):
    """A read size that ends exactly on the inflated end (and, for BGZF, on a block border): the final read hands out
    0 bytes with `last` set, the case in which the pinned reader must not add a second newline."""
    data = _text(2 * bgzf.BLOCK_INPUT)
    plain, gz, multi, bg = _write_sources(tmp_path, data)
    path = {"gzip": gz, "multi": multi, "bgzf": bg}[kind]
    for n in (bgzf.BLOCK_INPUT, 2 * bgzf.BLOCK_INPUT, bgzf.BLOCK_INPUT // 2):
        got, flags = _drain(_GzipSource(str(path)), [n])
        assert b"".join(got) == data
        assert got[-1] == b"" and flags[-1] and not any(flags[:-1])
        assert all(len(g) == n for g in got[:-1])


def test_bgzf_block_table(tmp_path):
    data = _text(3 * bgzf.BLOCK_INPUT + 1234)
    bg = _write_sources(tmp_path, data)[3]
    src = _GzipSource(str(bg))
    sizes = [b[2] for b in src._blocks]
    assert sizes == [bgzf.BLOCK_INPUT] * 3 + [1234, 0]                     # the last member is the empty EOF block


def test_line_split_dispatcher_schema():
    import torch
    lib = os.path.join(os.path.dirname(nv.LIB_PATH), "libbnpk_torch.so")
    if not os.path.exists(lib):
        pytest.skip("libbnpk_torch.so not built")
    torch.ops.load_library(lib)
    assert str(torch.ops.bnpk.line_split.default._schema) == (
        "bnpk::line_split(Tensor chunk, int lines_per_entry, int field_line, int start_offset, int header_char, "
        "bool check_plus, int trim_cr, int max_rows) -> (Tensor, Tensor, Tensor)")
