"""Writers without a GPU: the NumPy writer oracle against the reference's goldens and the golden files, the BGZF
writer, the argument checks of the two C entry points and the compiled code of the format kernels."""
import ctypes
import gzip
import io
import os
import re
import shutil
import struct
import subprocess
import zlib

import numpy as np
import pytest

from bionumpy_b200 import _native as nv
from bionumpy_b200.io import bgzf
from bionumpy_b200.io.ingest import _bgzf_blocks
from oracle import bnp_oracle as oracle

import write_oracle as wo

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")

# tests/buffers.py:17-40 of the reference
FASTQ = "@headerishere\nCTTGTTGA\n+\n!!!!!!!!\n@anotherheader\nCGG\n+\n~~~\n"
FASTA = ">header\nCTTGTTGA\n>header2\nCGG\n"
MULTILINE = ">header\nCTTGCC\nGCCTCC\n>header2\nCCCCCC\nGGGCCC\nTTT\n"


def _u8(text):
    return np.frombuffer(text.encode() if isinstance(text, str) else text, dtype=np.uint8)


def _fasta_fields(chunk):
    _, starts, lens = oracle.two_line_fasta_split(chunk)
    return (oracle.gather_rows(chunk, starts[:, 0], lens[:, 0]), lens[:, 0],
            oracle.gather_rows(chunk, starts[:, 1], lens[:, 1]), lens[:, 1])


def _multiline_fields(chunk):
    _, hs, hl, flat, sl = oracle.multiline_fasta_split(np.append(chunk, np.uint8(ord(">"))))
    return oracle.gather_rows(chunk, hs, hl), hl, flat, sl


def test_oracle_reference_buffer_goldens():
    assert bytes(wo.write_fastq(_u8(FASTQ))) == FASTQ.encode()
    assert bytes(wo.fasta_text(*_fasta_fields(_u8(FASTA)))) == FASTA.encode()
    assert bytes(wo.multiline_fasta_text(*_multiline_fields(_u8(MULTILINE)), 6)) == MULTILINE.encode()


@pytest.mark.parametrize("fmt", ["fastq", "fasta"])
@pytest.mark.parametrize("chunked", [False, True])
def test_oracle_read_write_roundtrip(fmt, chunked):
    """test_io.py::test_read_write_roundtrip: each text x100, read (in 200-byte chunks), written back byte for byte."""
    text = (FASTQ if fmt == "fastq" else FASTA) * 100
    split, lpe = (oracle.fastq_split, 4) if fmt == "fastq" else (oracle.two_line_fasta_split, 2)
    out = []
    for chunk, _, _ in oracle.read_chunks(io.BytesIO(text.encode()), split, 200 if chunked else 1 << 20, lpe):
        out.append(wo.write_fastq(chunk) if fmt == "fastq" else wo.fasta_text(*_fasta_fields(chunk)))
    assert b"".join(bytes(o) for o in out) == text.encode()


def test_oracle_multiline_widths_and_empty_sequences():
    names = _u8("abc")
    text = wo.multiline_fasta_text(names, [1, 1, 1], _u8("ACGTACG"), [0, 3, 4], 2)
    assert bytes(text) == b">a\n>b\nAC\nG\n>c\nTA\nCG\n"
    assert bytes(wo.fasta_text(names, [1, 1, 1], _u8("ACG"), [0, 3, 0])) == b">a\n\n>b\nACG\n>c\n\n"


def test_oracle_big_fastq(big_fq_bytes):
    assert np.array_equal(wo.write_fastq(big_fq_bytes), big_fq_bytes)


def test_oracle_saccer3_at_width_50():
    with gzip.open(os.path.join(GOLDEN, "sacCer3.fa.gz")) as f:
        data = np.frombuffer(f.read(), dtype=np.uint8)
    assert np.array_equal(wo.multiline_fasta_text(*_multiline_fields(data), 50), data)


def _members(raw):
    out, p = [], 0
    while p < len(raw):
        assert raw[p:p + 4] == b"\x1f\x8b\x08\x04"
        xlen = struct.unpack_from("<H", raw, p + 10)[0]
        assert raw[p + 12:p + 14] == b"BC"
        size = struct.unpack_from("<H", raw, p + 16)[0] + 1
        out.append(raw[p:p + size])
        p += size
    return out


def test_bgzf_writer_roundtrip_blocks_and_eof():
    rng = np.random.default_rng(1)
    text = bytes(rng.integers(0, 256, 300000, dtype=np.uint8)) + b"ACGT" * 200000   # incompressible + compressible
    sink = io.BytesIO()
    w = bgzf.BgzfWriter(_Keep(sink))
    for a in range(0, len(text), 77777):
        w.write(text[a:a + 77777])
    w.close()
    raw = sink.getvalue()
    assert gzip.decompress(raw) == text
    members = _members(raw)
    assert all(len(m) <= 65536 for m in members)
    assert members[-1] == bgzf.EOF_BLOCK and len(bgzf.EOF_BLOCK) == 28
    blocks = _bgzf_blocks(memoryview(raw))
    assert blocks is not None and sum(b[2] for b in blocks) == len(text)
    assert b"".join(zlib.decompress(raw[o:o + s], wbits=-15) for o, s, _ in blocks) == text
    assert max(b[2] for b in blocks) == bgzf.BLOCK_INPUT


def test_bgzf_writer_appends_members(tmp_path):
    path = tmp_path / "x.gz"
    for part in (b"first\n", b"second\n"):
        with bgzf.BgzfWriter(open(path, "ab")) as w:
            w.write(part)
    raw = path.read_bytes()
    assert gzip.decompress(raw) == b"first\nsecond\n"
    assert _bgzf_blocks(memoryview(raw)) is not None
    if shutil.which("zcat"):
        assert subprocess.run(["zcat", str(path)], capture_output=True).stdout == b"first\nsecond\n"


class _Keep:
    """A file object whose close() keeps the bytes readable."""

    def __init__(self, f):
        self._f = f

    def write(self, b):
        return self._f.write(b)

    def flush(self):
        pass

    def close(self):
        pass


def _fields(n_fields=3, starts=1, lens=1, base=0):
    arr = (nv.Field * 3)()
    for i in range(n_fields):
        arr[i] = nv.Field(base or None, 0, starts or None, lens or None, None)
    return arr


def _offsets_call(lib, fmt=nv.FMT_FASTQ, width=1, n=0, fields=None, status=1):
    fields = _fields() if fields is None else fields
    z = ctypes.c_void_p(0)
    return lib.bnpk_format_offsets(fmt, width, n, ctypes.cast(fields, ctypes.c_void_p) if fields is not False else z,
                                   z, ctypes.c_void_p(status), z, 0, z)


def _records_call(lib, fmt=nv.FMT_FASTQ, width=1, n=0, fields=None, begin=0, end=0, out=0):
    fields = _fields() if fields is None else fields
    z = ctypes.c_void_p(0)
    return lib.bnpk_format_records(fmt, width, n, ctypes.cast(fields, ctypes.c_void_p) if fields is not False else z,
                                   z, begin, end, ctypes.c_void_p(out), z)


@pytest.mark.parametrize("call", [_offsets_call, _records_call])
def test_entry_point_argument_errors(call):
    """Every bad argument is BNPK_E_BADARG, returned before any device work (so also without a GPU); an empty range
    of bnpk_format_records returns 0 without touching the device."""
    lib = nv.load_library()
    if call is _records_call:
        for fmt, width in ((nv.FMT_FASTQ, 1), (nv.FMT_FASTA, 0), (nv.FMT_FASTA_WRAPPED, 1), (nv.FMT_FASTA_WRAPPED, 4096)):
            assert call(lib, fmt=fmt, width=width) == 0
        assert call(lib, fmt=nv.FMT_FASTA, n=5, fields=_fields(2)) == 0         # FASTA reads no quality field
    for kwargs in (dict(fmt=3), dict(fmt=-1), dict(fmt=nv.FMT_FASTA_WRAPPED, width=0),
                   dict(fmt=nv.FMT_FASTA_WRAPPED, width=-5), dict(fields=False), dict(n=5, fields=_fields(2)),
                   dict(n=5, fields=_fields(3, starts=0)), dict(n=5, fields=_fields(3, lens=0)),
                   dict(fmt=nv.FMT_FASTA, n=5, fields=_fields(1))):
        assert call(lib, **kwargs) == nv.E_BADARG, kwargs
    if call is _records_call:
        assert call(lib, begin=5, end=5) == 0
        for kwargs in (dict(begin=5, end=4), dict(begin=-1, end=4), dict(begin=0, end=16, out=0),
                       dict(begin=0, end=16, out=1, n=0)):
            assert call(lib, **kwargs) == nv.E_BADARG, kwargs


def test_format_kernels_are_sm90a_code_without_stack():
    tool = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(tool):
        pytest.skip("cuobjdump not available")
    out = subprocess.run([tool, "-res-usage", nv.LIB_PATH], capture_output=True, text=True).stdout
    usage = {m.group(1): (int(m.group(2)), int(m.group(3)))
             for m in re.finditer(r"Function (\S+):\s*REG:(\d+) STACK:(\d+)", out)}
    fmt = {n: v for n, v in usage.items() if re.search(r"format_kernel|format_offsets_kernel", n)}
    assert len(fmt) == 3, sorted(fmt)                 # offsets scan + format kernel in write and check mode
    for name, (regs, stack) in fmt.items():
        assert stack == 0 and regs <= 96 and "rows_kernel" not in name, (name, regs, stack)
