"""Both chunk readers against the reference reader (tests/reader_oracle.py): PinnedFileReader, which bnp.open takes for
.fq / .fa and their .gz forms (pread, single-stream and multi-member gzip, block-parallel BGZF), and CudaFileReader
built directly over open() / gzip.open().  Every chunk's bytes, record count and '\\r' decision, and every record's
fields, must equal the oracle's, at every min_chunk_size up to a small file's length and at sizes that make a
source's last read return 0 bytes."""
import gzip

import numpy as np
import pytest
import torch

import reader_oracle as ro
from bionumpy_b200.io import bgzf

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def bnp():
    import bionumpy_b200
    return bionumpy_b200


def make_text(seed, n, lpe, maxlen=40, crlf=False, final_newline=True, truncate=0, long_record=0):
    rng = np.random.default_rng(seed)
    eol = b"\r\n" if crlf else b"\n"
    lines = []
    for r in range(n):
        L = long_record if (long_record and r == n // 2) else int(rng.integers(0, maxlen + 1))
        seq = bytes(rng.choice(np.frombuffer(b"ACGT", dtype=np.uint8), size=L).tolist())
        if lpe == 4:
            lines += [b"@r%d x" % r, seq, b"+", bytes(rng.integers(33, 74, size=L).astype(np.uint8).tolist())]
        else:
            lines += [b">r%d x" % r, seq]
    if truncate:
        lines = lines[:-truncate]
    text = b"".join(l + eol for l in lines)
    return text if final_newline else text[:-1]


def write(tmp_path, text, kind, lpe):
    suffix = ".fq" if lpe == 4 else ".fa"
    path = tmp_path / (f"{kind}{suffix}" + ("" if kind == "plain" else ".gz"))
    if kind == "plain":
        path.write_bytes(text)
    elif kind == "gzip":
        path.write_bytes(gzip.compress(text))
    elif kind == "multi":
        cut = [0, len(text) // 3, len(text) // 2 + 1, len(text)]
        path.write_bytes(b"".join(gzip.compress(text[a:b]) for a, b in zip(cut[:-1], cut[1:])))
    else:
        with open(path, "wb") as f:
            w = bgzf.BgzfWriter(f)
            w.write(text)
            w.close()
    return str(path)


def fmt(lpe):
    return ro.FASTQ if lpe == 4 else ro.FASTA


def buffer_type(bnp, lpe):
    from bionumpy_b200.io.buffers import CudaFastQBuffer, CudaTwoLineFastaBuffer
    return CudaFastQBuffer if lpe == 4 else CudaTwoLineFastaBuffer


def open_both(bnp, path, lpe):
    from bionumpy_b200.io.ingest import PinnedFileReader
    from bionumpy_b200.io.parser import CudaFileReader, NpDataclassReader
    pinned = bnp.open(path, buffer_type=buffer_type(bnp, lpe))
    assert isinstance(pinned._reader, PinnedFileReader)
    raw = gzip.open(path) if path.endswith(".gz") else open(path, "rb")
    generic = NpDataclassReader(CudaFileReader(raw, buffer_type(bnp, lpe)))
    return pinned, generic


def expected_cr(data, lpe):
    lines = data.split(b"\n")
    return len(lines[0]) > 0 and any(lines[i].endswith(b"\r") for i in range(0, min(lpe * lpe, len(lines) - 1), lpe))


def rows(field, add=0):
    r = field.raw() if hasattr(field, "raw") else field
    flat = (r.ravel().cpu().numpy().astype(np.uint8) + np.uint8(add)).tobytes()
    ends = np.cumsum(r.lengths.cpu().numpy())
    return [flat[a:b] for a, b in zip(np.concatenate([[0], ends[:-1]]).tolist(), ends.tolist())]


def records_of(entries, lpe):
    cols = [rows(entries.name), rows(entries.sequence)] + ([rows(entries.quality, 33)] if lpe == 4 else [])    # QualityEncoding: byte - 33
    return list(zip(*cols))


def oracle_records(chunk, lpe):
    return [(r[0], r[1], r[3]) if lpe == 4 else r for r in chunk.records]


def compare(bnp, path, text, lpe, sizes, records_for=()):
    """Both readers at every min_chunk_size in `sizes`: each chunk's bytes, n_lines_read and '\\r' flag; the records
    themselves for the sizes in `records_for`."""
    from bionumpy_b200.io.ingest import PinnedFileReader
    for m in sizes:
        want = ro.read_chunks(text, m, **fmt(lpe))
        # A file without a final newline whose size is a multiple of m: the pinned reader knows its read was the last
        # one and gives the record its newline at once, so the last record joins the chunk before it (the reference
        # loses it; the generic reader gives it a chunk of its own).  Compared as one piece.
        joined = text[-1:] != b"\n" and len(text) % m == 0
        for reader in open_both(bnp, path, lpe):
            with reader:
                got = []
                for buff in reader._reader.read_chunks(m):
                    got.append((bytes(buff._data.cpu().numpy()), reader._reader.n_lines_read, buff._cr))
                name = (m, type(reader._reader).__name__)
                if joined and isinstance(reader._reader, PinnedFileReader):
                    assert b"".join(g[0] for g in got) == b"".join(c.data for c in want), name
                    assert got[-1][1] == want[-1].n_lines_read, name
                    continue
                assert [g[0] for g in got] == [c.data for c in want], name
                assert [g[1] for g in got] == [c.n_lines_read for c in want], name
                assert [g[2] for g in got] == [expected_cr(c.data, lpe) for c in want], name
        if m in records_for:
            flat = [r for c in want for r in oracle_records(c, lpe)]
            for reader in open_both(bnp, path, lpe):
                with reader:
                    got = [records_of(c, lpe) for c in reader.read_chunks(m)]
                if joined and isinstance(reader._reader, PinnedFileReader):
                    assert [r for c in got for r in c] == flat, m
                else:
                    assert got == [oracle_records(c, lpe) for c in want], m


VARIANTS = {                       # name: make_text keywords
    "lf": {}, "crlf": dict(crlf=True), "no_final_nl": dict(final_newline=False),
    "crlf_no_final_nl": dict(crlf=True, final_newline=False),
    "trunc1": dict(truncate=1), "trunc2": dict(truncate=2), "trunc3": dict(truncate=3),
}


@pytest.mark.parametrize("kind", ["plain", "gzip", "multi", "bgzf"])
@pytest.mark.parametrize("lpe", [4, 2])
def test_every_chunk_size_of_a_small_file(bnp, tmp_path, kind, lpe):
    text = make_text(1, 24 if lpe == 4 else 40, lpe)
    assert 1000 < len(text) < 2600
    path = write(tmp_path, text, kind, lpe)
    n = len(text)
    sizes = range(1, n + 2) if (kind, lpe) == ("plain", 4) else \
        sorted(set(range(1, 17)) | set(range(17, n + 2, 53)) | {d for d in range(1, n + 1) if n % d == 0} | {n - 1, n})
    compare(bnp, path, text, lpe, sizes, records_for=(1, 16, n // 3, n))


@pytest.mark.parametrize("variant", list(VARIANTS))
@pytest.mark.parametrize("kind", ["plain", "gzip", "bgzf"])
@pytest.mark.parametrize("lpe", [4, 2])
def test_variants(bnp, tmp_path, variant, kind, lpe):
    """CRLF, no final newline and truncated files, at chunk sizes that divide the file (the last read returns 0
    bytes) and at others."""
    if lpe == 2 and variant == "trunc3":
        pytest.skip("two-line FASTA has only one line to cut from a record")
    text = make_text(2, 12, lpe, maxlen=30, **VARIANTS[variant])
    path = write(tmp_path, text, kind, lpe)
    n = len(text)
    divisors = [d for d in range(1, n + 1) if n % d == 0]
    sizes = sorted(set([d for d in divisors if d >= 8] + [17, 50, n - 1, n + 1]))
    compare(bnp, path, text, lpe, sizes, records_for=(17, divisors[len(divisors) // 2], n))


def test_truncated_tail_at_a_zero_byte_last_read(bnp, tmp_path):
    """A file whose tail ends in '\\n' one line short of an entry, read at a chunk size that divides it: the final
    read of a gzip source returns 0 bytes; the tail must not become a record."""
    for lpe, tail in ((4, b"@r\nAC\n+\n"), (2, b">r\n")):
        body = make_text(3, 10, lpe)
        text = body + tail
        for kind in ("plain", "gzip", "multi", "bgzf"):
            path = write(tmp_path, text, kind, lpe)
            sizes = [d for d in range(4, len(text) + 1) if len(text) % d == 0]
            compare(bnp, path, text, lpe, sizes, records_for=sizes[-3:])
            for m in sizes:
                with bnp.open(path, buffer_type=buffer_type(bnp, lpe)) as f:
                    assert sum(len(c) for c in f.read_chunks(m)) == 10


@pytest.mark.parametrize("kind", ["plain", "gzip", "bgzf"])
def test_record_longer_than_the_chunk(bnp, tmp_path, kind):
    text = make_text(4, 9, 4, long_record=5000, truncate=0)
    path = write(tmp_path, text, kind, 4)
    compare(bnp, path, text, 4, [7, 100, 999, 4096, len(text)], records_for=[100])


def test_large_file_chunk_sizes(bnp, tmp_path):
    text = make_text(5, 2400, 4, maxlen=120)
    assert 250_000 < len(text) < 400_000
    n = len(text)
    divisors = [d for d in range(2, 40) if n % d == 0]
    sizes = [n // d for d in divisors] + [bgzf.BLOCK_INPUT, 2 * bgzf.BLOCK_INPUT, bgzf.BLOCK_INPUT - 1, 300000, n]
    for kind in ("plain", "gzip", "bgzf"):
        path = write(tmp_path, text, kind, 4)
        compare(bnp, path, text, 4, sizes, records_for=(300000,))


def test_max_chunk_size_below_one_record(bnp, tmp_path):
    text = make_text(6, 5, 4, long_record=300)
    for kind in ("plain", "gzip"):
        path = write(tmp_path, text, kind, 4)
        with pytest.raises(ro.ReaderNoCompleteEntry):
            ro.read_chunks(text, 64, max_chunk_size=200, **ro.FASTQ)
        for reader in open_both(bnp, path, 4):
            with reader, pytest.raises(Exception, match="No complete entry found"):
                for _ in reader.read_chunks(64, 200):
                    pass


@pytest.mark.parametrize("where", ["first_chunk", "later_chunk", "first_entry_of_a_chunk"])
@pytest.mark.parametrize("kind", ["plain", "gzip"])
def test_format_exception_line_numbers(bnp, tmp_path, where, kind):
    from bionumpy_b200.io.exceptions import FormatException
    valid = b"@header\nacgtt\n+\n!!!!!\n"
    for bad, line in ((b"@header\nactg\n-\n!!!!\n", 2), (b"header\nactg\n+\n!!!!\n", 0)):
        if where == "first_chunk":
            text, m = valid * 3 + bad + valid, 1000
        elif where == "later_chunk":
            text, m = valid * 100 + bad + valid, 200
        else:
            text, m = valid * 10 + bad + valid * 3, len(valid) * 10           # the bad entry opens the second chunk
        with pytest.raises(ro.ReaderFormatError) as e:
            ro.read_chunks(text, m, **ro.FASTQ)
        path = write(tmp_path, text, kind, 4)
        for reader in open_both(bnp, path, 4):
            with reader, pytest.raises(FormatException) as g:
                for _ in reader.read_chunks(m):
                    pass
            assert g.value.line_number == e.value.line_number, (where, type(reader._reader).__name__)


def test_read_and_count_entries(bnp, tmp_path):
    for variant in ("lf", "crlf", "no_final_nl", "trunc2"):
        text = make_text(7, 40, 4, **VARIANTS[variant])
        want = [(r[0], r[1], r[3]) for r in ro.read_all(text, **ro.FASTQ)]
        for kind in ("plain", "gzip", "bgzf"):
            path = write(tmp_path, text, kind, 4)
            for reader in open_both(bnp, path, 4):
                with reader:
                    assert records_of(reader.read(), 4) == want, (variant, kind)
            assert bnp.count_entries(path) == len(want)


def test_two_readers_on_two_streams(bnp, tmp_path):
    text = make_text(8, 3000, 4, maxlen=80)
    path = write(tmp_path, text, "bgzf", 4)
    want = ro.read_chunks(text, 20000, **ro.FASTQ)
    streams = [torch.cuda.Stream(), torch.cuda.Stream()]
    readers = [bnp.open(path), bnp.open(path)]
    got = [[], []]
    its = [r._reader.read_chunks(20000) for r in readers]
    done = [False, False]
    while not all(done):
        for i in (0, 1):
            if done[i]:
                continue
            with torch.cuda.stream(streams[i]):
                b = next(its[i], None)
                if b is None:
                    done[i] = True
                else:
                    got[i].append(bytes(b._data.cpu().numpy()))
    for r in readers:
        r.close()
    assert got[0] == got[1] == [c.data for c in want]
