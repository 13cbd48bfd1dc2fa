"""NumPy restatement of the reference's BED parsing and interval sequences, for the interval tests (the package never
imports it).

Each function cites the reference lines (bionumpy/ unless noted) it follows."""
import numpy as np

TEXT, INT, INT_OR_DOT, STRAND, SKIP = "text", "int", "int_or_dot", "strand", "skip"
BED = (TEXT, INT, INT)
BED6 = (TEXT, INT, INT, TEXT, INT_OR_DOT, STRAND)
_COMPLEMENTS = {"A": "T", "G": "C", "C": "G", "T": "A", "N": "N"}


class Fault(Exception):
    """FormatException(line_number) of the reference."""

    def __init__(self, line, what):
        super().__init__(f"line {line}: {what}")
        self.line = line


def str_to_int(text):
    """io/strops.py:86-110 for one field: an optional '-' or '+', then digits.  More than 18 digits is a fault here
    (int64 holds every 18-digit number; the reference wraps)."""
    sign = 1
    if text[:1] in (b"-", b"+"):
        sign, text = (-1 if text[:1] == b"-" else 1), text[1:]
    if not text or len(text) > 18 or not all(48 <= c <= 57 for c in text):
        raise ValueError(text)
    return sign * int(text)


def parse_delimited(chunk, kinds):
    """DelimitedBuffer.from_raw_buffer + _get_buffer_extractor + _modify_for_carriage_return + get_data
    (io/delimited_buffers.py:52-83,203-232,278-316) for the columns `kinds` names.  Returns (size, columns): size = bytes
    up to and including the last newline, a column per kind (text: list of bytes; int/int_or_dot: int64 array; strand:
    uint8 codes '+' 0, '-' 1, '.' 2; skip: None).  Raises Fault(line) at the first bad line."""
    chunk = bytes(chunk)
    size = chunk.rfind(b"\n") + 1
    if size == 0:
        raise EOFError("no complete line")
    lines = chunk[:size - 1].split(b"\n")
    n_fields = lines[0].count(b"\t") + 1                           # _get_n_fields: the first line's delimiters
    cr = lines[0].endswith(b"\r")                                   # _modify_for_carriage_return: decided by line 0
    columns = [[] for _ in kinds]
    for i, line in enumerate(lines):
        if cr and line.endswith(b"\r"):
            line = line[:-1]
        fields = line.split(b"\t")
        if len(fields) != n_fields:
            raise Fault(i, "irregular number of delimiters")
        if len(fields) < len(kinds):
            raise Fault(i, "too few columns")
        for c, kind in enumerate(kinds):
            f = fields[c]
            if kind == TEXT:
                columns[c].append(f)
            elif kind in (INT, INT_OR_DOT):
                if kind == INT_OR_DOT and f == b".":             # str_to_int_with_missing, io/strops.py:69-83
                    columns[c].append(0)
                    continue
                try:
                    columns[c].append(str_to_int(f))
                except ValueError:
                    raise Fault(i, "not an integer") from None
            elif kind == STRAND:
                if f not in (b"+", b"-", b"."):                     # StrandEncoding, encodings/alphabet_encoding.py:120
                    raise Fault(i, "not a strand")
                columns[c].append(b"+-.".index(f))
    out = []
    for kind, col in zip(kinds, columns):
        if kind == SKIP:
            out.append(None)
        elif kind == TEXT:
            out.append(col)
        elif kind == STRAND:
            out.append(np.array(col, dtype=np.uint8))
        else:
            out.append(np.array(col, dtype=np.int64))
    return size, out


def read_delimited(data, kinds, min_chunk_size):
    """NumpyFileReader.read_chunks (io/parser.py:96-171) over `parse_delimited`: chunks of at least min_chunk_size bytes
    cut after their last newline, the tail carried over; a fault's line is made global with the lines read before
    (parser.py:139-143).  Returns the columns of the whole file, concatenated."""
    if data and not data.endswith(b"\n"):
        data = data + b"\n"
    pos, n_lines, parts = 0, 0, []
    while pos < len(data):
        end = pos + min_chunk_size
        while True:
            piece = data[pos:end]
            if b"\n" in piece or end >= len(data):
                break
            end += min_chunk_size
        try:
            size, cols = parse_delimited(piece, kinds)
        except Fault as e:
            raise Fault(e.line + n_lines, str(e)) from None
        parts.append(cols)
        n_lines += data[pos:pos + size].count(b"\n")
        pos += size
    out = []
    for c, kind in enumerate(kinds):
        cols = [p[c] for p in parts]
        if kind == SKIP:
            out.append(None)
        elif kind == TEXT:
            out.append([f for col in cols for f in col])
        else:
            out.append(np.concatenate(cols) if cols else np.zeros(0, dtype=np.int64))
    return out


def read_fai(text):
    """read_index, io/indexed_fasta.py:13-31."""
    out = {}
    for line in text.splitlines():
        name, rlen, offset, lenc, lenb = line.split("\t")[:5]
        out[name.split()[0]] = {"rlen": int(rlen), "offset": int(offset), "lenc": int(lenc), "lenb": int(lenb)}
    return out


def interval_sequences(file_bytes, index, chromosomes, starts, stops):
    """IndexedFasta.get_interval_sequences, io/indexed_fasta.py:178-206: per interval, seek to the first base, read
    through the last, and delete the line ends.  Intervals are checked first (the package raises ValueError where the
    reference would read neighbouring bytes).  Returns (flat uint8, lengths)."""
    f = np.frombuffer(bytes(file_bytes), dtype=np.uint8)
    pieces, lengths = [], []
    for chromosome, start, stop in zip(chromosomes, starts, stops):
        idx = index[chromosome]
        if not 0 <= start <= stop <= idx["rlen"]:
            raise ValueError((chromosome, start, stop))
        lenb, lenc = idx["lenb"], idx["lenc"]
        start_row, start_mod = start // lenc, start % lenc
        start_offset = start_row * lenb + start_mod
        stop_row = stop // lenc
        stop_offset = stop_row * lenb + stop % lenc
        lengths.append(stop_offset - start_offset - (stop_row - start_row))
        tmp = f[idx["offset"] + start_offset: idx["offset"] + stop_offset]
        tmp = np.delete(tmp, [lenb * (j + 1) - 1 - start_mod for j in range(stop_row - start_row)])
        pieces.append(tmp)
    flat = np.concatenate(pieces) if pieces else np.zeros(0, dtype=np.uint8)
    return flat, np.array(lengths, dtype=np.int64)


def complement_table(alphabet=None):
    """sequence/dna.py:13-34: the complement as a 256-entry table; ASCII text (alphabet None) knows A, C, G, T, N in
    upper case and maps every other byte to 0."""
    table = np.zeros(256, dtype=np.uint8)
    if alphabet is None:
        for k, v in _COMPLEMENTS.items():
            table[ord(k)] = ord(v)
    else:
        for i, c in enumerate(alphabet):
            table[i] = alphabet.index(_COMPLEMENTS[c])
    return table


def strand_specific_sequences(sequence, starts, stops, strands, alphabet=None):
    """get_strand_specific_sequences, sequence/dna.py:68-88: sequence[start:stop], reverse-complemented where the
    strand is '-'.  Returns a list of uint8 rows."""
    seq = np.asarray(sequence, dtype=np.uint8)
    table = complement_table(alphabet)
    out = []
    for a, b, s in zip(starts, stops, strands):
        if not 0 <= a <= b <= seq.size:
            raise ValueError((a, b))
        row = seq[a:b]
        out.append(table[row[::-1]] if s in ("-", 1) else row.copy())
    return out


def _digits(values, width):
    """Right-aligned decimal digits of non-negative ints: (bytes [N, width], number of digits [N])."""
    v = np.asarray(values, dtype=np.int64)
    n_dig = np.maximum(1, np.floor(np.log10(np.maximum(v, 1))).astype(np.int64) + 1)
    pw = 10 ** np.arange(width - 1, -1, -1, dtype=np.int64)
    return (48 + (v[:, None] // pw) % 10).astype(np.uint8), n_dig


def synthetic_bed(n, chromosomes, seed=0, max_start=10 ** 8, max_len=1000):
    """A BED text of n lines "chrom \\t start \\t stop \\n" built without a Python loop per line, and its truth:
    (bytes, chromosome index int64[n], start int64[n], stop int64[n])."""
    rng = np.random.default_rng(seed)
    names = [c.encode() for c in chromosomes]
    ci = rng.integers(0, len(names), n)
    start = rng.integers(0, max_start, n)
    stop = start + rng.integers(0, max_len, n)
    w = 19
    ds, ns = _digits(start, w)
    de, ne = _digits(stop, w)
    name_w = max(len(b) for b in names)
    name_tab = np.zeros((len(names), name_w), dtype=np.uint8)
    for i, b in enumerate(names):
        name_tab[i, :len(b)] = np.frombuffer(b, dtype=np.uint8)
    name_len = np.array([len(b) for b in names])[ci]
    rows = np.concatenate([name_tab[ci], np.full((n, 1), 9, np.uint8), ds, np.full((n, 1), 9, np.uint8), de,
                           np.full((n, 1), 10, np.uint8)], axis=1)
    col = np.arange(rows.shape[1])
    keep = np.concatenate([col[None, :name_w] < name_len[:, None], np.ones((n, 1), bool),
                           col[None, :w] >= (w - ns)[:, None], np.ones((n, 1), bool),
                           col[None, :w] >= (w - ne)[:, None], np.ones((n, 1), bool)], axis=1)
    return rows[keep].tobytes(), ci, start, stop
