"""Time track profiles on seeded synthetic data on hg38: the fused column mean of equal-length windows
(RunsRaggedArray.mean(axis=0) on bnpk_runs_column_sum / bnpk_track_f64_column_sum) against the materialised path on
the same inputs (every position gathered by bnpk_runs_extract, reshaped, torch's mean), alternating in one call; then
get_windows, and the summit profile of the goldens end to end.  Prints one JSON line; --check also compares the fused
and materialised results (integer sums exactly, float sums to 1e-12 relative, and two fused calls bit for bit).

    python tools/profile_bench.py --check"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bionumpy_b200 as bnp  # noqa: E402
from bionumpy_b200 import _native as nv, ops  # noqa: E402
from bionumpy_b200.arithmetics.intervals import (FloatRunLengthArray, GenomicRunLengthArray,  # noqa: E402
                                                 RunsRaggedArray, coverage_runs)
from bionumpy_b200.genomic_data.genome import GenomicLocation  # noqa: E402

GOLDEN = os.path.join(ROOT, "tests", "golden")


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()
    return out[0] if out else torch.cuda.get_device_name(0)


def timed(fn, repeat):
    """Median milliseconds of fn() between CUDA events, after one warm-up call."""
    fn()
    times = []
    for _ in range(repeat):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        times.append(a.elapsed_time(b))
    return float(np.median(times))


def contig_positions(gen, genome, n, margin):
    """n random global positions at least ``margin`` from every contig border, contigs drawn by size."""
    sizes = np.array(list(genome._sizes.values()), dtype=np.int64)
    offsets = np.array([genome._offsets[k] for k in genome._sizes], dtype=np.int64)
    ok = sizes > 2 * margin + 1
    p = np.where(ok, sizes, 0) / np.where(ok, sizes, 0).sum()
    c = gen.choice(sizes.size, n, p=p)
    local = (gen.random(n) * (sizes[c] - 2 * margin - 1)).astype(np.int64) + margin
    return c, offsets[c] + local, local


def materialised_mean(track, q, width):
    """The parent's path: every position gathered, reshaped, torch's mean."""
    n = q.numel()
    offsets = torch.arange(n + 1, dtype=torch.int64, device=q.device) * width
    flat = track._cast(ops.runs_extract(track._events, track._values64(), q, offsets, n * width))
    return flat.reshape(n, width).to(torch.float64).mean(0)


def compare(name, track, q, width, n_rev, repeat, check, results):
    dev = q.device
    gen = torch.Generator(device="cpu").manual_seed(7)
    rev = (torch.rand(q.numel(), generator=gen) < 0.5).to(dev) if n_rev else None
    windows = RunsRaggedArray(track, q, q + width, rev)
    plain = RunsRaggedArray(track, q, q + width)
    is_float = isinstance(track, FloatRunLengthArray)
    kernel = ops.track_f64_column_sum if is_float else ops.runs_column_sum
    values = track._values.contiguous() if is_float else track._values64()
    rev8 = None if rev is None else rev.to(torch.uint8)
    t_kernel = timed(lambda: kernel(track._events, values, q, width, rev8), repeat)
    fused, mat = [], []
    for _ in range(repeat):           # alternating, same inputs
        fused.append(timed(lambda: windows.mean(axis=0), 1))
        mat.append(timed(lambda: materialised_mean(track, q, width), 1))
    n = q.numel()
    row = {"case": name, "rows": n, "width": width, "kernel_ms": round(t_kernel, 4),
           "fused_mean_ms": round(float(np.median(fused)), 4), "materialised_mean_ms": round(float(np.median(mat)), 4),
           "gpositions_per_s_kernel": round(n * width / t_kernel / 1e6, 2),
           "materialised_bytes": n * width * 8}
    if check:
        a = plain.sum(axis=0)
        b = plain.sum(axis=0)
        ref_mean = materialised_mean(track, q, width)
        got_mean = plain.mean(axis=0)
        if is_float:
            ok = torch.equal(a.view(torch.int64), b.view(torch.int64))
            ok = ok and bool(torch.allclose(got_mean, ref_mean, rtol=1e-12, atol=0, equal_nan=True))
        else:
            offsets = torch.arange(n + 1, dtype=torch.int64, device=dev) * width
            flat = ops.runs_extract(track._events, track._values64(), q, offsets, n * width)
            ok = torch.equal(a, flat.reshape(n, width).sum(0)) and torch.equal(a, b)
            ok = ok and bool(torch.allclose(got_mean, ref_mean, rtol=1e-12, atol=0))
        row["check"] = bool(ok)
    results.append(row)


def summit_profile():
    genome = bnp.Genome.from_file(os.path.join(GOLDEN, "hg38.chrom.sizes"))
    peaks = bnp.open(os.path.join(GOLDEN, "ctcf_chr21-22.bed.gz"), buffer_type=bnp.io.NarrowPeakBuffer).read()
    summits = genome.get_locations(bnp.LocationEntry(peaks.chromosome, peaks.start + peaks.summit)).sorted()
    windows = summits.get_windows(flank=200)
    reads = genome.read_intervals(os.path.join(GOLDEN, "ctcf_chr21-22_every6th.bam"), stranded=True)
    out = {s: reads[reads.strand == s].get_pileup()[windows].mean(axis=0) for s in "+-"}
    torch.cuda.synchronize()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reads", type=int, default=10_000_000)
    ap.add_argument("--windows", type=int, default=1_000_000)
    ap.add_argument("--repeat", type=int, default=5)
    ap.add_argument("--check", action="store_true")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "profile_bench needs a CUDA device"
    dev = torch.device("cuda:0")
    gen = np.random.default_rng(0)
    genome = bnp.Genome.from_file(os.path.join(GOLDEN, "hg38.chrom.sizes"))
    # 10 M stranded 150-bp reads, their pileup as global runs
    _, r_start, _ = contig_positions(gen, genome, args.reads, 200)
    g0 = torch.from_numpy(r_start).to(dev)
    runs, values, _ = coverage_runs(g0, g0 + 150, genome.size, nv.PILEUP_COUNT)
    pileup = GenomicRunLengthArray(runs, values, genome.size)
    # a MACS2-shaped float64 track: fold-enrichment-like values on the same runs
    signal = FloatRunLengthArray(runs, values.to(torch.float64) * 0.731 + 0.0113, genome.size)
    results = []
    _, w_pos, _ = contig_positions(gen, genome, args.windows, 600)
    q = torch.from_numpy(w_pos - 500).to(dev)
    compare("pileup_1M_x_1001_stranded", pileup, q, 1001, True, args.repeat, args.check, results)
    compare("float_track_1M_x_1001_stranded", signal, q, 1001, True, args.repeat, args.check, results)
    _, w_pos, _ = contig_positions(gen, genome, 1000, 60_000)
    compare("pileup_1000_x_100kb", pileup, torch.from_numpy(w_pos - 50_000).to(dev), 100_000, False, args.repeat,
            args.check, results)
    # get_windows of 1 M locations
    c, g_pos, local = contig_positions(gen, genome, args.windows, 600)
    name_index = {n: i for i, n in enumerate(genome._name_table()[0])}
    ids = torch.from_numpy(np.array([name_index[n] for n in genome._sizes], dtype=np.int64)[c]).to(dev)
    strand = torch.from_numpy(gen.integers(0, 2, args.windows).astype(np.uint8)).to(dev)
    loc = GenomicLocation(ids, torch.from_numpy(g_pos).to(dev), torch.from_numpy(local).to(dev), genome, strand)
    t_windows = timed(lambda: loc.get_windows(flank=500), args.repeat)
    summit_profile()
    t0 = time.perf_counter()
    summit_profile()
    t_summit = (time.perf_counter() - t0) * 1e3
    print(json.dumps({"card": card(), "runs": int(values.numel()), "cases": results,
                      "get_windows_1M_ms": round(t_windows, 4), "summit_profile_goldens_ms": round(t_summit, 2)}))
    if args.check and not all(r["check"] for r in results):
        sys.exit(1)


if __name__ == "__main__":
    main()
