"""A plain Python restatement of BAM reading (SAM spec 4.2) and a minimal BAM/BGZF writer for synthetic files.  Test
infrastructure only: it never imports the package.

  parse_bam(data)      : header and records of gzip-inflated BAM bytes, by a struct walk over block_size prefixes
  parse_sam(path)      : the records of a SAM text file, in the same dict form
  record_bytes(rec)    : one record serialised (block_size included); header_bytes, bgzf and write_bam build files
  reference_length, bed6_rows, fastq_text : the values the package derives from the records"""
import gzip
import struct
import zlib

import numpy as np

SEQ = "=ACMGRSVTWYHKDBN"
CIGAR = "MIDNSHP=X"
CONSUMING = set("MDN=X")


def parse_header(data):
    """(names, lengths, size of the header) of inflated BAM bytes."""
    assert data[:4] == b"BAM\1"
    l_text = struct.unpack_from("<i", data, 4)[0]
    p = 8 + l_text
    n_ref = struct.unpack_from("<i", data, p)[0]
    p += 4
    names, lengths = [], []
    for _ in range(n_ref):
        l_name = struct.unpack_from("<i", data, p)[0]
        names.append(data[p + 4:p + 3 + l_name].decode())
        lengths.append(struct.unpack_from("<i", data, p + 4 + l_name)[0])
        p += 8 + l_name
    return names, lengths, p


def parse_record(data, p):
    """The record at offset p and the offset after it."""
    block_size, ref_id, pos, l_name, mapq, _bin, n_cigar, flag, l_seq, next_ref, next_pos, tlen = \
        struct.unpack_from("<iiiBBHHHiiii", data, p)
    q = p + 36
    name = data[q:q + l_name - 1]
    q += l_name
    words = struct.unpack_from(f"<{n_cigar}I", data, q)
    q += 4 * n_cigar
    packed = data[q:q + (l_seq + 1) // 2]
    q += (l_seq + 1) // 2
    codes = [(packed[i // 2] >> (0 if i % 2 else 4)) & 15 for i in range(l_seq)]
    qual = data[q:q + l_seq]
    q += l_seq
    end = p + 4 + block_size
    return dict(ref_id=ref_id, pos=pos, mapq=mapq, flag=flag, name=bytes(name), cigar=[(w & 15, w >> 4) for w in words],
                seq=codes, qual=bytes(qual), next_ref_id=next_ref, next_pos=next_pos, tlen=tlen,
                aux=bytes(data[q:end])), end


def parse_bam(data):
    """(names, lengths, records, record offsets) of inflated BAM bytes."""
    names, lengths, p = parse_header(data)
    records, offsets = [], []
    while p < len(data):
        offsets.append(p)
        rec, p = parse_record(data, p)
        records.append(rec)
    assert p == len(data)
    return names, lengths, records, offsets


def read_bam(path):
    with open(path, "rb") as f:
        return parse_bam(gzip.decompress(f.read()))


def chromosome(rec, names):
    return "*" if rec["ref_id"] < 0 else names[rec["ref_id"]]


def cigar_text(cigar):
    return "".join(f"{n}{CIGAR[op]}" for op, n in cigar) or "*"


def seq_text(codes):
    return "".join(SEQ[c] for c in codes)


def parse_sam(path):
    """The alignment lines of a SAM file: name, flag, chromosome, 0-based position, mapq, cigar, sequence and quality
    (phred values) of each."""
    out = []
    for line in open(path):
        if line.startswith("@"):
            continue
        f = line.rstrip("\n").split("\t")
        out.append(dict(name=f[0].encode(), flag=int(f[1]), chromosome=f[2], pos=int(f[3]) - 1, mapq=int(f[4]),
                        cigar=f[5], seq="" if f[9] == "*" else f[9],
                        qual=b"" if f[10] == "*" else bytes(ord(c) - 33 for c in f[10])))
    return out


def reference_length(cigar):
    return sum(n for op, n in cigar if CIGAR[op] in CONSUMING)


def bed6_rows(records, names, placed_only=False):
    """(chromosome, start, stop, name, score, strand) of every record (of every placed record)."""
    return [(chromosome(r, names), r["pos"], r["pos"] + reference_length(r["cigar"]), r["name"].decode(), r["mapq"],
             "-" if r["flag"] & 16 else "+") for r in records if not placed_only or r["ref_id"] >= 0]


def fastq_text(records):
    """The records as FASTQ: the stored quality + 33 (0xFF wraps to 0x20, as a uint8 sum does)."""
    return b"".join(b"@" + r["name"] + b"\n" + seq_text(r["seq"]).encode() + b"\n+\n" +
                    bytes((q + 33) & 255 for q in r["qual"]) + b"\n" for r in records)


# ---- writing ------------------------------------------------------------------------------------------------------
def record_bytes(ref_id=0, pos=0, name=b"r", mapq=0, flag=0, cigar=(), seq=(), qual=None, next_ref_id=-1, next_pos=-1,
                 tlen=0, aux=b"", block_size=None, l_name=None, l_seq=None, n_cigar=None):
    """One BAM record.  The keyword overrides (block_size, l_name, l_seq, n_cigar) write a field as given even when it
    disagrees with the data, to build malformed records."""
    seq = list(seq)
    qual = bytes([255] * len(seq)) if qual is None else bytes(qual)
    name_z = bytes(name) + b"\0"
    packed = bytearray((len(seq) + 1) // 2)
    for i, c in enumerate(seq):
        packed[i // 2] |= c << (0 if i % 2 else 4)
    body = struct.pack("<iiBBHHHiiii", ref_id, pos, len(name_z) if l_name is None else l_name, mapq, 4680,
                       len(cigar) if n_cigar is None else n_cigar, flag, len(seq) if l_seq is None else l_seq,
                       next_ref_id, next_pos, tlen)
    body += name_z + b"".join(struct.pack("<I", n << 4 | op) for op, n in cigar) + bytes(packed) + qual + aux
    return struct.pack("<i", len(body) if block_size is None else block_size) + body


def header_bytes(names, lengths, text=b""):
    out = b"BAM\1" + struct.pack("<i", len(text)) + text + struct.pack("<i", len(names))
    for n, ln in zip(names, lengths):
        out += struct.pack("<i", len(n) + 1) + n.encode() + b"\0" + struct.pack("<i", ln)
    return out


def bgzf(data, block=65280, level=1):
    """BGZF (SAM spec 4.1): members of at most `block` inflated bytes with the BC extra field, then the EOF block."""
    out = bytearray()
    for a in range(0, len(data), block):
        piece = data[a:a + block]
        c = zlib.compressobj(level, zlib.DEFLATED, -15)
        raw = c.compress(piece) + c.flush()
        out += b"\x1f\x8b\x08\x04\0\0\0\0\0\xff\x06\0BC\x02\0" + struct.pack("<H", len(raw) + 25)
        out += raw + struct.pack("<II", zlib.crc32(piece) & 0xFFFFFFFF, len(piece))
    out += b"\x1f\x8b\x08\x04\0\0\0\0\0\xff\x06\0BC\x02\0\x1b\0\x03\0\0\0\0\0\0\0\0\0"
    return bytes(out)


def random_records(rng, n, n_ref, read_len=(0, 300), aux_len=(0, 40), unmapped=0.0):
    """n records with every base code and cigar op, names of 1..40 bytes, odd and even lengths and aux bytes."""
    out = []
    for i in range(n):
        l_seq = int(rng.integers(*read_len))
        n_cigar = int(rng.integers(0, 4))
        ref = -1 if rng.random() < unmapped else int(rng.integers(0, n_ref))
        out.append(dict(ref_id=ref, pos=int(rng.integers(-1, 1 << 20)),
                        name=bytes(rng.integers(33, 127, int(rng.integers(1, 41))).astype(np.uint8)),
                        mapq=int(rng.integers(0, 256)), flag=int(rng.integers(0, 1 << 16)),
                        cigar=[(int(rng.integers(0, 9)), int(rng.integers(0, 1 << 20))) for _ in range(n_cigar)],
                        seq=[int(x) for x in rng.integers(0, 16, l_seq)],
                        qual=bytes(rng.integers(0, 256, l_seq).astype(np.uint8)),
                        aux=bytes(rng.integers(0, 256, int(rng.integers(*aux_len))).astype(np.uint8))))
    return out


def write_bam(path, names, lengths, records, text=b"", block=65280):
    """A BGZF BAM file of the records (dicts as parse_record gives, or raw record bytes); returns the inflated bytes."""
    data = header_bytes(names, lengths, text) + b"".join(
        r if isinstance(r, bytes) else record_bytes(**r) for r in records)
    with open(path, "wb") as f:
        f.write(bgzf(data, block))
    return data
