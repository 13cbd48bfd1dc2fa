"""Plain-Python restatement of GTF/GFF reading, attribute values, feature selection and spliced transcript sequences,
for the annotation tests (the package never imports it).  It follows bionumpy/datatypes/gtf.py,
io/delimited_buffers.py:486-595 (GTFBuffer, GFFBuffer, DelimitedBufferWithInernalComments) and sequence/genes.py,
with the rules the package documents where those differ: one value per row and key matched whole, or a fault;
exons joined in ascending start order."""
import gzip

FIELDS = ("chromosome", "source", "feature_type", "start", "stop", "score", "strand", "phase", "atributes")
KEYS = {"gene": ("gene_id",), "transcript": ("gene_id", "transcript_id"),
        "exon": ("gene_id", "transcript_id", "exon_id")}
STRANDS = {b"+": 0, b"-": 1, b".": 2}
_COMP = {ord(a): ord(b) for a, b in zip("ACGTNacgtn", "TGCANtgcan")}


class Fault(Exception):
    """FormatException(line_number) of the package."""

    def __init__(self, line, what):
        super().__init__(f"line {line}: {what}")
        self.line = line
        self.what = what


class BadBase(Exception):
    def __init__(self, offset):
        super().__init__(f"bad base at flat offset {offset}")
        self.offset = offset


def read_file(path):
    with (gzip.open(path) if str(path).endswith(".gz") else open(path, "rb")) as f:
        return f.read()


def split_header(data):
    """DelimitedBuffer.read_header: the leading '#' lines are the header; returns the rest."""
    i = 0
    while i < len(data) and data[i:i + 1] == b"#":
        j = data.find(b"\n", i)
        i = len(data) if j < 0 else j + 1
    return data[i:]


def parse(chunk, gff):
    """The rows of a chunk without header: (rows, size).  A row is a dict of the nine fields (text as bytes with its
    chunk offset in ``<field>_at``, start and stop int, strand a code), plus ``line``, its line in the chunk.  GFF drops
    every line that starts with '#'.  Raises Fault(line) for a line whose tab count differs from the first row's, a bad
    integer or a bad strand; line counts every line of the chunk, comments included."""
    size = chunk.rfind(b"\n") + 1
    lines, pos, rows = [], 0, []
    for line in chunk[:size].split(b"\n")[:-1]:
        lines.append((pos, line))
        pos += len(line) + 1
    kept = [(i, p, l) for i, (p, l) in enumerate(lines) if not (gff and l[:1] == b"#")]
    if not kept:
        return rows, size
    n_tabs = kept[0][2].count(b"\t")
    cr = kept[0][2].endswith(b"\r")
    for i, p, line in kept:
        if cr and line.endswith(b"\r"):
            line = line[:-1]
        fields = line.split(b"\t")
        if len(fields) - 1 != n_tabs:
            raise Fault(i, "irregular number of delimiters")
        if len(fields) < 9:
            raise Fault(i, "too few columns")
        row, at = {"line": i}, p
        for name, f in zip(FIELDS, fields):
            if name in ("start", "stop"):
                digits = f[1:] if f[:1] in (b"+", b"-") else f
                if not digits or len(digits) > 18 or not digits.isdigit():
                    raise Fault(i, "bad integer")
                row[name] = -int(digits) if f[:1] == b"-" else int(digits)
            elif name == "strand":
                if f not in STRANDS:
                    raise Fault(i, "bad strand")
                row[name] = STRANDS[f]
            else:
                row[name] = f
                row[name + "_at"] = at
            at += len(f) + 1
        rows.append(row)
    return rows, size


def read(path_or_bytes, gff):
    data = path_or_bytes if isinstance(path_or_bytes, bytes) else read_file(path_or_bytes)
    data = split_header(data)
    if data and not data.endswith(b"\n"):
        data += b"\n"
    return parse(data, gff)[0]


def attribute_values(text, keys, gff):
    """{key: (value offset, value length)} of the keys found in one attribute column; the first attribute with a key
    wins.  GTF: ``key value`` or ``key "value"`` (';' inside quotes kept, unquoted values trimmed of trailing spaces);
    GFF: ``key=value`` as written."""
    keys = [k.encode() if isinstance(k, str) else k for k in keys]
    found, i, n = {}, 0, len(text)
    sep = ord("=") if gff else ord(" ")
    while i < n:
        while i < n and text[i] == 32:
            i += 1
        if i >= n:
            break
        if text[i] == 59:
            i += 1
            continue
        ks = i
        while i < n and text[i] not in (59, sep):
            i += 1
        key = text[ks:i]
        if i >= n or text[i] == 59:         # an attribute without a value
            i += 1
            continue
        i += 1
        if gff:
            end = text.find(b";", i)
            end = n if end < 0 else end
            value, i = (i, end - i), end + 1
        else:
            while i < n and text[i] == 32:
                i += 1
            if i < n and text[i] == 34:
                close = text.find(b'"', i + 1)
                if close < 0:
                    value, i = (i + 1, n - i - 1), n
                else:
                    value = (i + 1, close - i - 1)
                    semi = text.find(b";", close + 1)
                    i = n if semi < 0 else semi + 1
            else:
                semi = text.find(b";", i)
                end = n if semi < 0 else semi
                e = end
                while e > i and text[e - 1] == 32:
                    e -= 1
                value, i = (i, e - i), end + 1
        if key in keys and key not in found:
            found[key] = value
    return {k.decode(): v for k, v in found.items()}


def select(rows, feature, gff, keys=None):
    """get_genes / get_transcripts / get_exons: the rows of one feature type with their attribute values (bytes).
    Raises Fault(index of the row in ``rows``, key) for a selected row without a key."""
    keys = KEYS[feature] if keys is None else keys
    out = []
    for r, row in enumerate(rows):
        if row["feature_type"] != feature.encode():
            continue
        values = attribute_values(row["atributes"], keys, gff)
        for k in keys:
            if k not in values:
                raise Fault(r, k)
        new = dict(row)
        for k in keys:
            s, n = values[k]
            new[k] = row["atributes"][s:s + n]
        out.append(new)
    return out


def transcripts(exons):
    """Runs of consecutive exons with equal transcript_id, in file order: [(transcript_id, strand, [exons])]."""
    out = []
    for e in exons:
        if out and out[-1][0] == e["transcript_id"]:
            out[-1][2].append(e)
        else:
            out.append((e["transcript_id"], e["strand"], [e]))
    return out


def reverse_complement(seq):
    return bytes(_COMP.get(c, c) for c in reversed(seq))


def transcript_sequences(exons, fetch):
    """[(transcript_id, sequence)]: each transcript's exons sorted by start (descending on '-', stably), each fetched
    with fetch(chromosome, start, stop) and reverse-complemented on '-', joined, then upper-cased.  A byte other than
    ACGTN in either case raises BadBase with its flat offset in the joined output."""
    out, flat = [], 0
    for tid, strand, group in transcripts(exons):
        minus = strand == 1
        ordered = sorted(group, key=lambda e: -e["start"] if minus else e["start"])
        parts = [fetch(e["chromosome"], e["start"], e["stop"]) for e in ordered]
        seq = b"".join(reverse_complement(p) if minus else p for p in parts)
        for j, c in enumerate(seq):
            if chr(c).upper() not in "ACGTN":
                raise BadBase(flat + j)
        flat += len(seq)
        out.append((tid, seq.upper()))
    return out


def reference_order_sequences(exons, fetch):
    """sequence/genes.py of the reference: exons joined in file order, the whole reverse-complemented on '-'."""
    out = []
    for tid, strand, group in transcripts(exons):
        seq = b"".join(fetch(e["chromosome"], e["start"], e["stop"]) for e in group)
        out.append((tid, (reverse_complement(seq) if strand == 1 else seq).upper()))
    return out
