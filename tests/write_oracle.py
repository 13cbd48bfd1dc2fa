"""The writers restated with NumPy: records (names, sequences, qualities as flat bytes + row lengths) -> file text.
Each function follows the reference's construction step for step.  Test infrastructure only; the package never imports
it."""
import numpy as np

from oracle import bnp_oracle as oracle


def _ragged_rows(flat, lens):
    ends = np.cumsum(np.asarray(lens, dtype=np.int64))
    return np.split(np.asarray(flat, dtype=np.uint8), ends[:-1]) if len(lens) else []


def join_fields(fields, line_offsets, header, n_lines_per_entry):
    """OneLineBuffer.join_fields (io/one_line_buffer.py:119-134): line i of an entry is line_offsets[i] bytes of room
    (the header char on line 0), the field, and '\\n'.  ``fields``: [(flat, lens)] per line."""
    field_lengths = np.stack([np.asarray(l, dtype=np.int64) for _, l in fields], axis=1)   # :121
    line_lengths = field_lengths + 1                                                        # :122
    line_lengths += np.asarray(line_offsets[:len(fields)], dtype=np.int64)                 # :123-124
    buf = np.zeros(int(line_lengths.sum()), dtype=np.uint8)                                # :125-127
    ends = np.cumsum(line_lengths.ravel())
    starts = ends - line_lengths.ravel()
    step = n_lines_per_entry
    for i, (flat, lens) in enumerate(fields):                                              # :130-131
        idx = oracle.ragged_indices(starts[i::step] + line_offsets[i], lens)
        buf[idx] = np.asarray(flat, dtype=np.uint8)
    buf[starts[0::step]] = ord(header)                                                     # :132
    buf[ends - 1] = ord("\n")                                                              # :133
    return buf


def fastq_text(names, name_lens, seqs, seq_lens, quals, qual_lens):
    """FastQBuffer.from_data / join_fields (io/fastq_buffer.py:47-61): the '+' line is a field of one '+' per entry;
    qualities are QualityEncoding.decode'd: byte = v + 33."""
    n = len(name_lens)
    plus = (np.full(n, ord("+"), dtype=np.uint8), np.ones(n, dtype=np.int64))
    q = (np.asarray(quals, dtype=np.int64) + 33).astype(np.uint8)
    return join_fields([(names, name_lens), (seqs, seq_lens), plus, (q, qual_lens)], (1, 0, 0, 0), "@", 4)


def fasta_text(names, name_lens, seqs, seq_lens):
    """TwoLineFastaBuffer (io/one_line_buffer.py:185-192) through join_fields."""
    return join_fields([(names, name_lens), (seqs, seq_lens)], (1, 0), ">", 2)


def multiline_fasta_text(names, name_lens, seqs, seq_lens, width):
    """MultiLineFastaBuffer.from_data (io/multiline_buffer.py:67-86).  An entry with an empty sequence is written as its
    header line alone (the reference assigns that entry's last-line length to its header line instead)."""
    name_lens = np.asarray(name_lens, dtype=np.int64)
    seq_lens = np.asarray(seq_lens, dtype=np.int64)
    n_lines = (seq_lens + width - 1) // width                                             # :70 (0 lines for Ls = 0)
    last_length = (seq_lens - 1) % width + 1                                               # :71
    line_lengths = np.full(int(np.sum(n_lines)) + n_lines.size, width + 1, dtype=np.int64)  # :72
    entry_starts = np.insert(np.cumsum(n_lines + 1), 0, 0)                                 # :73
    has_seq = n_lines > 0
    line_lengths[entry_starts[1:][has_seq] - 1] = last_length[has_seq] + 1                 # :75
    line_lengths[entry_starts[:-1]] = name_lens + 2                                        # :74
    ends = np.cumsum(line_lengths)
    starts = ends - line_lengths
    buf = np.zeros(int(line_lengths.sum()), dtype=np.uint8)
    buf[oracle.ragged_indices(starts[entry_starts[:-1]] + 1, name_lens)] = np.asarray(names, dtype=np.uint8)  # :78
    buf[starts[entry_starts[:-1]]] = ord(">")                                              # :79
    idxs = np.delete(np.arange(line_lengths.size), entry_starts[:-1])                      # :80
    buf[oracle.ragged_indices(starts[idxs], line_lengths[idxs] - 1)] = np.asarray(seqs, dtype=np.uint8)  # :81-83
    buf[ends - 1] = ord("\n")                                                              # :84
    return buf


def read_fastq(chunk):
    """(names, name_lens, seqs, seq_lens, quals, qual_lens) of a FASTQ chunk with the oracle's reader."""
    chunk = np.asarray(chunk, dtype=np.uint8)
    _, starts, lens = oracle.fastq_split(chunk)
    g = lambda c: (oracle.gather_rows(chunk, starts[:, c], lens[:, c]), lens[:, c])
    (n, nl), (s, sl), (q, ql) = g(0), g(1), g(3)
    return n, nl, s, sl, q.astype(np.int64) - 33, ql


def write_fastq(chunk):
    return fastq_text(*read_fastq(chunk))
