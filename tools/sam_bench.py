"""SAM reading on the GPU: kernel times of the line split, bnpk_sam_columns, bnpk_cigar_count and bnpk_cigar_unpack
(CUDA events over repeated launches), the columns kernel's share of the HBM bound, the CIGAR kernels on long-read
CIGARs, and bnp.open(...).read() and read_intervals(...).get_pileup() end to end for a .sam, a .sam.gz and a .bam of
the same records.  --check compares a subset against tests/sam_oracle.py.  Prints one JSON object (and writes it to
--out) with the card's name and power limit.

The kernel input is --records lines of 150 bases with realistic tags (NM, MD, AS, XS, RG), 95 % 150M CIGARs and the
rest soft-clipped, deleted or inserted, generated from a seed by vectorised numpy code as 100 k distinct lines
repeated on the device."""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import bam_oracle as bo                       # noqa: E402
import sam_oracle as so                       # noqa: E402
import bionumpy_b200 as bnp                   # noqa: E402
from bionumpy_b200 import ops                 # noqa: E402
from bionumpy_b200.io.sam import SAMBuffer    # noqa: E402

HBM = 3.35e12                                 # H100 SXM data sheet, bytes/s
NAMES = [f"chr{i}" for i in range(1, 23)]
SIZE = 1 << 28
READ = 150


def _s(a):
    return np.asarray(a).astype(str).astype(np.bytes_)


def _rows_text(m):
    """uint8[n, w] -> n bytes strings of w bytes."""
    return np.ascontiguousarray(m).view(f"S{m.shape[1]}").reshape(-1)


def sam_lines(n, seed=0):
    """n SAM lines (bytes array, no newline) of READ bases: names r<i>, flags of paired reads, positions on NAMES,
    95 % 150M and 5 % soft-clipped, deleted or inserted CIGARs, and five tags."""
    rng = np.random.default_rng(seed)
    cat = np.char.add
    a = rng.integers(1, 50, n)
    kind = rng.choice(4, n, p=[0.95, 0.02, 0.02, 0.01])
    cigar = np.where(kind == 0, b"150M", b"")
    cigar = np.where(kind == 1, cat(cat(_s(a), b"S"), cat(_s(READ - a), b"M")), cigar)
    cigar = np.where(kind == 2, cat(cat(cat(_s(a), b"M"), cat(_s(a % 7 + 1), b"D")), cat(_s(READ - a), b"M")), cigar)
    cigar = np.where(kind == 3, cat(cat(cat(_s(a), b"M"), cat(_s(a % 5 + 1), b"I")),
                                    cat(_s(READ - a - a % 5 - 1), b"M")), cigar)
    pos = rng.integers(1, SIZE - 1000, n)
    seq = _rows_text(np.frombuffer(b"ACGT", dtype=np.uint8)[rng.integers(0, 4, (n, READ))])
    qual = _rows_text(rng.integers(33, 75, (n, READ)).astype(np.uint8))
    cols = [cat(b"r", _s(np.arange(n))), _s(rng.choice([99, 147, 83, 163, 0, 16], n)),
            np.array([x.encode() for x in NAMES])[rng.integers(0, len(NAMES), n)], _s(pos), _s(rng.integers(0, 61, n)),
            cigar, np.full(n, b"="), _s(pos + rng.integers(100, 400, n)), _s(rng.integers(-500, 500, n)), seq, qual,
            cat(b"NM:i:", _s(rng.integers(0, 5, n))), np.full(n, b"MD:Z:150"), cat(b"AS:i:", _s(rng.integers(100, 151, n))),
            cat(b"XS:i:", _s(rng.integers(0, 100, n))), np.full(n, b"RG:Z:grp1")]
    line = cols[0]
    for c in cols[1:]:
        line = cat(cat(line, b"\t"), c)
    return line


def long_cigars(n, n_ops, seed=1):
    """n CIGAR strings of about n_ops ops each, every op letter, as text rows on the device."""
    rng = np.random.default_rng(seed)
    ops_ = np.frombuffer(b"MIDNSHP=X", dtype=np.uint8)[rng.integers(0, 9, n * n_ops)]
    lens = _s(rng.integers(1, 10000, n * n_ops))
    text = np.char.add(lens, ops_.view("S1"))
    rows = [b"".join(text[i * n_ops:(i + 1) * n_ops].tolist()) for i in range(n)]
    lens_ = [len(r) for r in rows]
    base = torch.frombuffer(bytearray(b"".join(rows)), dtype=torch.uint8).cuda()
    starts = torch.tensor(np.concatenate([[0], np.cumsum(lens_)[:-1]]), dtype=torch.int64).cuda()
    return base, starts, torch.tensor(lens_, dtype=torch.int32).cuda()


def events(fn, reps):
    fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps


def wall(fn, reps=3):
    fn()
    torch.cuda.synchronize()
    t = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        t.append(time.perf_counter() - t0)
    return min(t)


def check(lines):
    """The fields, CIGARs and rows of the lines against the oracle."""
    data = b"".join(x + b"\n" for x in lines)
    recs, fault = so.read_sam(data)
    assert fault is None
    e = SAMBuffer.from_raw_buffer(data).get_data()
    for f in so.FIELDS:
        v = getattr(e, f)
        if f in ("flag", "position", "mapq", "next_position", "length"):
            assert v.cpu().tolist() == [r[f] for r in recs], f
        else:
            raw = v.ravel().raw().cpu().numpy().tobytes()
            ends = np.cumsum(v.lengths.cpu().numpy())
            assert [raw[a:b] for a, b in zip(np.concatenate([[0], ends[:-1]]), ends)] == [r[f] for r in recs], f
    op, length = bnp.alignments.parse_cigar(e.cigar)
    flat_op, flat_len = op.ravel().raw().cpu().tolist(), length.ravel().cpu().tolist()
    want = [x for r in recs for x in so.parse_cigar(r["cigar"])]
    assert list(zip(flat_op, flat_len)) == want
    b = bnp.alignments.alignment_to_interval(e)
    assert b.stop.cpu().tolist() == [row[2] for row in so.bed6_rows(recs)]
    return len(recs)


def bam_of(lines):
    """BAM records (bytes) of SAM lines, for the end-to-end comparison with the BAM reader."""
    recs, _ = so.read_sam(b"".join(x + b"\n" for x in lines))
    codes = {c: i for i, c in enumerate(bo.SEQ)}
    out = []
    for r in recs:
        out.append(bo.record_bytes(ref_id=NAMES.index(r["chromosome"].decode()), pos=r["position"] - 1,
                                   name=r["name"], mapq=r["mapq"], flag=r["flag"], cigar=so.parse_cigar(r["cigar"]),
                                   seq=[codes[chr(c)] for c in r["sequence"]], qual=[q - 33 for q in r["quality"]],
                                   next_ref_id=NAMES.index(r["chromosome"].decode()), next_pos=r["next_position"] - 1,
                                   tlen=r["length"]))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--records", type=int, default=10_000_000)
    ap.add_argument("--e2e-records", type=int, default=1_000_000)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--check", action="store_true")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()[0]
    res = {"gpu": gpu}
    t0 = time.perf_counter()
    base = sam_lines(100_000)
    res["generate_100k_lines_s"] = time.perf_counter() - t0
    if args.check:
        res["checked_lines"] = check(base[:3000].tolist()) + check(sam_lines(2000, seed=7).tolist())
    one = np.frombuffer(b"".join(x + b"\n" for x in base.tolist()), dtype=np.uint8)
    reps = max(1, args.records // len(base))
    d = torch.from_numpy(one.copy()).cuda().repeat(reps)
    n = len(base) * reps
    res["records"], res["line_bytes"] = n, d.numel()
    res["split_ms"] = events(lambda: ops.line_split(d, 1, 0, 0, ord("@"), False, 0, max_rows=n), args.reps)
    starts, lens, _ = ops.line_split(d, 1, 0, 0, ord("@"), False, 0, max_rows=n)
    res["columns_ms"] = events(lambda: ops.sam_columns(d, starts, lens), args.reps)
    res["columns_hbm_share"] = d.numel() / HBM / (res["columns_ms"] / 1e3)
    fields, st = ops.sam_columns(d, starts, lens)
    assert ops.read_status(st).fault is None
    c_starts, c_lens = fields[4], fields[5].to(torch.int32)
    res["cigar_count_ms"] = events(lambda: ops.cigar_count(d, c_starts, c_lens), args.reps)
    counts, _, _ = ops.cigar_count(d, c_starts, c_lens)
    offsets = ops.row_offsets(counts)
    total = int(offsets[-1])
    res["cigar_ops"] = total
    res["cigar_unpack_ms"] = events(lambda: ops.cigar_unpack(d, c_starts, c_lens, offsets, total), args.reps)
    del d, starts, lens, fields, c_starts, c_lens, counts, offsets
    torch.cuda.empty_cache()
    lb, ls, ll = long_cigars(20_000, 2000)
    counts, _, _ = ops.cigar_count(lb, ls, ll)
    offsets = ops.row_offsets(counts)
    total = int(offsets[-1])
    res["long_rows"], res["long_ops"], res["long_text_bytes"] = ls.numel(), total, lb.numel()
    res["long_count_ms"] = events(lambda: ops.cigar_count(lb, ls, ll), args.reps)
    res["long_unpack_ms"] = events(lambda: ops.cigar_unpack(lb, ls, ll, offsets, total), args.reps)
    del lb, ls, ll, counts, offsets
    with tempfile.TemporaryDirectory() as tmp:
        sam, gz, bam, sizes = (os.path.join(tmp, x) for x in ("e.sam", "e.sam.gz", "e.bam", "g.sizes"))
        k = max(1, args.e2e_records // len(base))
        header = b"".join(b"@SQ\tSN:%s\tLN:%d\n" % (x.encode(), SIZE) for x in NAMES)
        text = header + one.tobytes() * k
        with open(sam, "wb") as fh:
            fh.write(text)
        with open(gz, "wb") as fh:
            fh.write(bo.bgzf(text))
        bo.write_bam(bam, NAMES, [SIZE] * len(NAMES), bam_of(base.tolist()) * k)
        del text
        with open(sizes, "w") as fh:
            fh.writelines(f"{x}\t{SIZE}\n" for x in NAMES)
        g = bnp.Genome.from_file(sizes)
        res["e2e_records"] = len(base) * k
        for name, path in (("sam", sam), ("sam_gz", gz), ("bam", bam)):
            res[f"{name}_file_bytes"] = os.path.getsize(path)
            res[f"{name}_read_s"] = wall(lambda: bnp.open(path).read().position)
            res[f"{name}_pileup_s"] = wall(lambda: g.read_intervals(path).get_pileup())
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
