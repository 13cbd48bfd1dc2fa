"""A plain Python restatement of SAM reading (SAM spec 1.4), the CIGAR grammar, the reference length and the interval
rows, and a writer of SAM text for generated records.  Test infrastructure only: it never imports the package.

  read_sam(data)        : (records, fault) of SAM bytes: the leading '@' lines are the header, every other line a
                          record of the 12 SAMEntry fields (bytes and ints), or the first fault as (line, column, kind)
  parse_cigar(text)     : [(op code, length)] of valid CIGAR text ("*" is []), None for invalid text
  reference_length, bed6_rows : the values alignment_to_interval and SAMIntervalBuffer give
  sam_line / bam_to_sam : SAM text of a record dict, and of the records of tests/bam_oracle.py"""
import re

FIELDS = ("name", "flag", "chromosome", "position", "mapq", "cigar", "next_chromosome", "next_position", "length",
          "sequence", "quality", "extra")
INTS = {1: "flag", 3: "position", 4: "mapq", 7: "next_position", 8: "length"}
BAD_COLUMNS, BAD_INT, BAD_CIGAR = 2, 3, 6          # the kinds of include/bnpk.h
CIGAR = "MIDNSHP=X"
CONSUMING = set("MDN=X")
_INT = re.compile(rb"[+-]?[0-9]{1,18}")
_CIGAR = re.compile(rb"\*|(?:[0-9]{1,9}[MIDNSHP=X])+")
_OP = re.compile(rb"([0-9]{1,9})([MIDNSHP=X])")


def split_lines(data):
    """(header lines, record lines) of SAM bytes; the record lines without their '\\n'.  A last line without one
    counts, as the reader adds a newline to a file that lacks it."""
    lines = data.split(b"\n")
    if lines and lines[-1] == b"":
        lines.pop()
    n = 0
    while n < len(lines) and lines[n].startswith(b"@"):
        n += 1
    return lines[:n], lines[n:]


def read_lines(lines):
    """(records, fault) of record lines.  When the first line ends in '\\r', a '\\r' that ends a line is dropped.
    fault = (line, column, kind) of the first line with fewer than 11 columns (column = its column count) or, in a line
    of 11 or more, the first FLAG, POS, MAPQ, PNEXT or TLEN that is not an optional sign and 1 to 18 digits."""
    cr = bool(lines) and lines[0].endswith(b"\r")
    records = []
    for i, line in enumerate(lines):
        if cr and line.endswith(b"\r"):
            line = line[:-1]
        cols = line.split(b"\t")
        if len(cols) < 11:
            return records, (i, len(cols), BAD_COLUMNS)
        for c in sorted(INTS):
            if not _INT.fullmatch(cols[c]):
                return records, (i, c, BAD_INT)
        rec = {f: (int(cols[c]) if c in INTS else cols[c]) for c, f in enumerate(FIELDS[:11])}
        rec["extra"] = b"\t".join(cols[11:])
        records.append(rec)
    return records, None


def read_sam(data):
    return read_lines(split_lines(data)[1])


def parse_cigar(text):
    """[(op code in MIDNSHP=X, length)] of CIGAR text, [] for "*", None when it is not "*" or ops of 1 to 9 digits and
    one of MIDNSHP=X."""
    text = bytes(text)
    if not _CIGAR.fullmatch(text):
        return None
    if text == b"*":
        return []
    return [(CIGAR.index(op.decode()), int(n)) for n, op in _OP.findall(text)]


def cigar_text(ops):
    return "".join(f"{n}{CIGAR[op]}" for op, n in ops) or "*"


def reference_length(ops):
    return sum(n for op, n in ops if CIGAR[op] in CONSUMING)


def first_bad_cigar(records):
    """The first record whose CIGAR is invalid, or None."""
    return next((i for i, r in enumerate(records) if parse_cigar(r["cigar"]) is None), None)


def bed6_rows(records, placed_only=False):
    """(chromosome, start, stop, name, score, strand) of every record (of every record whose RNAME is not '*'):
    start = POS - 1, stop = start + the reference length of the CIGAR."""
    out = []
    for r in records:
        if placed_only and r["chromosome"] == b"*":
            continue
        start = r["position"] - 1
        out.append((r["chromosome"].decode(), start, start + reference_length(parse_cigar(r["cigar"])),
                    r["name"].decode(), r["mapq"], "-" if r["flag"] & 16 else "+"))
    return out


def sam_line(rec):
    """One SAM line (no newline) of a record dict with the 12 fields (bytes or str text, ints)."""
    def b(v):
        return v if isinstance(v, bytes) else str(v).encode()
    line = b"\t".join(b(rec[f]) for f in FIELDS[:11])
    return line + (b"\t" + b(rec["extra"]) if rec.get("extra") else b"")


def bam_to_sam(names, records, header=b""):
    """SAM text of records parsed by tests/bam_oracle.py (aux fields are left out): the same names, flags, places,
    cigars, bases and qualities."""
    seq_codes = "=ACMGRSVTWYHKDBN"
    lines = [header.rstrip(b"\n")] if header else []
    for r in records:
        chrom = "*" if r["ref_id"] < 0 else names[r["ref_id"]]
        rnext = "*" if r["next_ref_id"] < 0 else "=" if r["next_ref_id"] == r["ref_id"] else names[r["next_ref_id"]]
        qual = r["qual"]
        lines.append(sam_line(dict(
            name=r["name"], flag=r["flag"], chromosome=chrom, position=r["pos"] + 1, mapq=r["mapq"],
            cigar=cigar_text(r["cigar"]), next_chromosome=rnext, next_position=r["next_pos"] + 1, length=r["tlen"],
            sequence="".join(seq_codes[c] for c in r["seq"]) or "*",
            quality="*" if not qual or qual[0] == 255 else bytes(q + 33 for q in qual))))
    return b"\n".join(lines) + b"\n"
