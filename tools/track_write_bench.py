"""Time tracks back into intervals and BED / bedGraph text on the device and print one JSON line (CUDA-event medians,
with the card and its power limit read by nvidia-smi in the same run), on hg38 with 10 M synthetic 150-bp intervals:
  from_track      GenomicIntervals.from_track of the intervals' mask
  get_data        GenomicArray.get_data of their pileup (a bedGraph of every run)
  format_bed3 / format_bdg
                  bnpk_delimited_format of 10 M BED3 lines and of the pileup's bedGraph lines (kernel alone), with the
                  HBM bound: the bytes the columns are read from plus the bytes written, at 3.35 TB/s
  write_bed / write_bed_gz / write_bdg
                  the README chain's writes end to end (host clock, file closed)
  oracle_100k     tests/delimited_write_oracle.py's dump_lines of 100 k BED3 lines on one CPU core.
--check compares the written files' bytes with the oracle's lines of the same rows, and the peaks read back with the
mask they came from (use a --threshold that leaves peaks at a small --n)."""
import argparse
import gzip
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

import bionumpy_b200 as bnp  # noqa: E402
from bionumpy_b200 import _native as nv  # noqa: E402
from bionumpy_b200.io.delimited import DelimitedText  # noqa: E402

HBM = 3.35e12


def median_ms(fn, iters):
    fn()
    times = []
    for _ in range(iters):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        times.append(a.elapsed_time(b))
    return float(np.median(times))


def host_ms(fn, iters):
    fn()
    times = []
    for _ in range(iters):
        torch.cuda.synchronize()
        t = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        times.append((time.perf_counter() - t) * 1e3)
    return float(np.median(times))


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip().splitlines()
    return out[0] if out else "unknown"


def synthetic(genome, n, rng):
    names = list(genome.chrom_sizes)
    sizes = np.array([genome.chrom_sizes[c] for c in names])
    c = np.sort(rng.choice(len(names), n, p=sizes / sizes.sum()))
    s = (rng.random(n) * (sizes[c] - 150)).astype(np.int64)
    return bnp.Interval([names[i] for i in c], s, s + 150)


def column_bytes(text):
    """Bytes the format kernel reads from the columns: the text bytes, 8 per integer and 4 + 8 per text row."""
    total = 8 * (len(text.offsets))
    for kind, data in text.columns:
        if kind == nv.COL_TEXT:
            total += int(data[2].to(torch.int64).sum()) + 12 * data[2].numel()
        else:
            total += data.numel() * data.element_size()
    return total


def rows_text(record):
    import delimited_write_oracle as wo
    cols = [("text", record.chromosome.tolist()), ("int", record.start.cpu().numpy()),
            ("int", record.stop.cpu().numpy())]
    if hasattr(record, "value"):
        cols.append(("int", record.value.to(torch.int64).cpu().numpy()))
    return wo.dump_lines(cols)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--n", type=int, default=10_000_000)
    ap.add_argument("--threshold", type=int, default=4, help="the README chain's peaks: pileup > threshold")
    ap.add_argument("--check", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("track_write_bench needs a CUDA device")
    import delimited_write_oracle as wo
    genome = bnp.Genome.from_file(os.path.join(ROOT, "tests", "golden", "hg38.chrom.sizes"))
    iv = genome.get_intervals(synthetic(genome, args.n, np.random.default_rng(1)))
    mask, pileup = iv.get_mask(), iv.get_pileup()
    res = {"card": card(), "n_intervals": args.n}
    res["from_track_ms"] = median_ms(lambda: bnp.GenomicIntervals.from_track(mask), args.iters)
    res["get_data_ms"] = median_ms(lambda: pileup.get_data(), args.iters)
    peaks_rec = bnp.GenomicIntervals.from_track(mask).get_data()
    bdg_rec = pileup.get_data()
    res["mask_rows"], res["bedgraph_rows"] = len(peaks_rec), len(bdg_rec)
    for name, rec in (("bed3", peaks_rec), ("bdg", bdg_rec)):
        text = DelimitedText(rec)
        out = torch.empty(text.size, dtype=torch.uint8, device="cuda")
        ms = median_ms(lambda: text.slice(0, text.size, out), args.iters)
        moved = column_bytes(text) + text.size
        res[f"format_{name}_lines"] = len(rec)
        res[f"format_{name}_ms"] = ms
        res[f"format_{name}_bytes"] = text.size
        res[f"format_{name}_hbm_fraction"] = moved / HBM / (ms * 1e-3)
    with tempfile.TemporaryDirectory() as tmp:
        peaks = bnp.GenomicIntervals.from_track(pileup > args.threshold).merged()
        paths = {k: os.path.join(tmp, f) for k, f in (("bed", "peaks.bed"), ("bed_gz", "peaks.bed.gz"),
                                                      ("bdg", "pileup.bdg"))}

        def write(path, data):
            bed = bnp.io.BedBuffer if ".bed" in path else None
            with bnp.open(path, "w", buffer_type=bed) as f:
                f.write(data)

        res["write_bed_ms"] = host_ms(lambda: write(paths["bed"], peaks_rec), max(args.iters // 2, 1))
        res["write_bed_gz_ms"] = host_ms(lambda: write(paths["bed_gz"], peaks_rec), max(args.iters // 5, 1))
        res["write_bdg_ms"] = host_ms(lambda: write(paths["bdg"], bdg_rec), max(args.iters // 2, 1))
        res["bed_bytes"], res["bdg_bytes"] = os.path.getsize(paths["bed"]), os.path.getsize(paths["bdg"])
        small = peaks_rec[torch.arange(min(100_000, len(peaks_rec)), device="cuda")]
        cols = [("text", small.chromosome.tolist()), ("int", small.start.cpu().numpy()),
                ("int", small.stop.cpu().numpy())]
        t = time.perf_counter()
        wo.dump_lines(cols)
        res["oracle_100k_ms"] = (time.perf_counter() - t) * 1e3
        if args.check:
            ok = open(paths["bed"], "rb").read() == rows_text(peaks_rec)
            ok &= gzip.open(paths["bed_gz"]).read() == open(paths["bed"], "rb").read()
            ok &= open(paths["bdg"], "rb").read() == rows_text(bdg_rec)
            ok &= int((genome.read_intervals(paths["bed"]).get_mask() ^ mask).sum()) == 0
            write(paths["bed"], peaks.get_data())
            ok &= int((genome.read_intervals(paths["bed"]).get_mask() ^ (pileup > args.threshold)).sum()) == 0
            res["check"] = bool(ok)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
