"""NumPy restatement of the reference's chunk reader for the one-line formats (FASTQ, two-line FASTA):
NumpyFileReader.read_chunk, _get_buffer and __add_newline_to_end (bionumpy/io/parser.py:96-206) over a byte string,
each chunk split by ``oracle.one_line_split``.  The package never imports this file.

One deliberate deviation is modelled by ``keep_unterminated_last``: when a file has no final newline and its size is a
multiple of ``min_chunk_size``, the reference's last read returns 0 bytes, ``_get_buffer`` returns None and the carried
tail, which holds the last record, is dropped.  Both readers of this package keep that record (True, the default);
False restates the reference exactly."""
from collections import namedtuple

import numpy as np

from oracle import bnp_oracle as o

Chunk = namedtuple("Chunk", "records n_lines_read data")    # data: the chunk's bytes, its complete entries

NEWLINE = 10
FASTQ = dict(lpe=4, header=ord("@"), line_offsets=(1, 0, 0, 0), check_plus=True)
FASTA = dict(lpe=2, header=ord(">"), line_offsets=(1, 0), check_plus=False)


class ReaderFormatError(Exception):
    def __init__(self, message, line_number):
        super().__init__(f"{message} (line {line_number})")
        self.line_number = line_number


class ReaderNoCompleteEntry(Exception):
    """read_chunk's ``Exception("No complete entry found")`` for a ``max_chunk_size`` below one entry."""


def split_records(chunk, lpe, header, line_offsets, check_plus):
    """(n_complete_bytes, n_lines, records) of one chunk: records are tuples of the lpe fields' bytes, '\\r' trimmed
    as the reference trims it.  Raises o.OracleIncompleteEntry / o.OracleFormatException like from_raw_buffer."""
    chunk = np.asarray(chunk, dtype=np.uint8)
    size, starts, lens = o.one_line_split(chunk, lpe, header, line_offsets, check_plus)
    raw = chunk.tobytes()
    recs = [tuple(raw[s:s + n] for s, n in zip(srow.tolist(), lrow.tolist())) for srow, lrow in zip(starts, lens)]
    return size, len(recs) * lpe, recs


def read_chunks(data: bytes, min_chunk_size, max_chunk_size=None, lpe=4, header=ord("@"), line_offsets=(1, 0, 0, 0),
                check_plus=True, keep_unterminated_last=True):
    """Every chunk the reference's read_chunks(min_chunk_size, max_chunk_size) yields for the file ``data``.

    Returns a list of Chunk(records, n_lines_read after the chunk, the chunk's bytes).  A FormatException becomes ReaderFormatError with the
    reference's global line number (line in the chunk + n_lines_read, parser.py:139-143)."""
    pos, n = 0, len(data)
    prepend = b""
    finished = False
    n_lines_read = 0
    out = []

    def get_buffer():                                             # parser.py:192-200
        nonlocal pos, finished
        a = data[pos:pos + min_chunk_size]
        pos += len(a)
        finished = len(a) < min_chunk_size
        if not a:
            return None
        if finished and a[-1] != NEWLINE:                         # parser.py:183-186
            a = a + b"\n"
        return a

    while not finished:                                           # read_chunks, parser.py:173-178
        temp = [prepend] if prepend else []
        found = None
        while found is None:
            chunk = get_buffer()
            if chunk is None:
                if keep_unterminated_last and temp and temp[-1] and temp[-1][-1] != NEWLINE:
                    chunk = b"\n"                                  # the deviation: the carried tail gets its newline
                    finished = True
                else:
                    return out
            temp.append(chunk)
            if max_chunk_size is not None and sum(len(c) for c in temp) > max_chunk_size:
                raise ReaderNoCompleteEntry("No complete entry found")
            joined = b"".join(temp)
            try:
                found = split_records(np.frombuffer(joined, dtype=np.uint8), lpe, header, line_offsets, check_plus)
            except o.OracleIncompleteEntry:
                if finished:
                    return out
            except o.OracleFormatException as e:
                raise ReaderFormatError(str(e), e.line_number + n_lines_read) from None
            temp = [joined]
        size, n_lines, recs = found
        prepend = b"" if finished else joined[size:]
        n_lines_read += n_lines
        out.append(Chunk(recs, n_lines_read, joined[:size]))
    return out


def read_all(data: bytes, **fmt):
    """Every record of the file (``read()``: one chunk of the whole file, parser.py:89-94)."""
    if not data:
        return []
    if data[-1] != NEWLINE:
        data = data + b"\n"
    try:
        return split_records(np.frombuffer(data, dtype=np.uint8), **fmt)[2]
    except o.OracleIncompleteEntry:
        return []
    except o.OracleFormatException as e:
        raise ReaderFormatError(str(e), e.line_number) from None


def plain_line_split(chunk):
    """lines_per_entry = 1 without validation: (n_complete_bytes, starts, lens) of every '\\n'-terminated line."""
    chunk = np.asarray(chunk, dtype=np.uint8)
    nl = np.flatnonzero(chunk == NEWLINE)
    starts = np.concatenate([[0], nl[:-1] + 1]).astype(np.int64) if nl.size else np.zeros(0, np.int64)
    return (int(nl[-1]) + 1 if nl.size else 0), starts, (nl - starts).astype(np.int64)
