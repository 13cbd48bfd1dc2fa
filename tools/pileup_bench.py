"""Pileups, masks, merges and run-length extraction on the device: kernel times against their HBM bound, the end-to-end
calls and the NumPy oracle.

    python tools/pileup_bench.py [--intervals 10000000] [--peaks 1000000] [--iters 10] [--check]

Workload 1: --intervals synthetic 150-bp intervals spread over the hg38 contigs without '_' (tests/golden/hg38.chrom.sizes):
the event sort (torch.sort) and bnpk_pileup_runs timed alone (CUDA-event medians), each with its HBM bound, then
GenomicIntervals.get_pileup, get_mask and merged end to end.  Workload 2: --peaks 100-bp peaks against that pileup:
the fused per-peak max (bnpk_runs_reduce) and the materialised extract.  Workload 3: the oracle on one CPU core for
100 k intervals.  Prints one JSON line with the card's name and power limit (read-only nvidia-smi query in the same
run); --check compares the runs and the per-peak maxima with the oracle (on 1 M intervals at most)."""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))

import bionumpy_b200 as bnp  # noqa: E402
from bionumpy_b200 import ops  # noqa: E402

from motif_bench import card, median_ms, HBM_BYTES_PER_S  # noqa: E402

import pileup_oracle as po  # noqa: E402


def bound(ms, n_bytes):
    b = n_bytes / HBM_BYTES_PER_S * 1e3
    return {"kernel_ms": round(ms, 4), "bytes": int(n_bytes), "bound_ms": round(b, 4), "share_of_bound": round(b / ms, 3)}


def synthetic(sizes, n, seed):
    """n 150-bp intervals, contigs in proportion to their size, sorted by contig and start."""
    names, offsets, total = po.genome_layout(sizes)
    rng = np.random.default_rng(seed)
    g = np.sort(rng.integers(0, total - 150, n))
    ends = np.array([offsets[c] + sizes[c] for c in names])
    cid = np.searchsorted(ends, g, side="right")
    start = g - np.array([offsets[c] for c in names])[cid]
    start = np.minimum(start, np.array([sizes[c] for c in names])[cid] - 150)
    return [names[i] for i in cid], start, start + 150


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--intervals", type=int, default=10_000_000)
    ap.add_argument("--peaks", type=int, default=1_000_000)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--check", action="store_true")
    args = ap.parse_args()
    sizes = po.read_sizes(open(os.path.join(ROOT, "tests", "golden", "hg38.chrom.sizes")).read())
    genome = bnp.Genome.from_dict(sizes, filter_function=lambda n: "_" not in n)
    chroms, start, stop = synthetic(sizes, args.intervals, 1)
    gi = genome.get_intervals(bnp.Interval(chroms, start, stop))
    n = len(gi)
    out = {"card": card(), "intervals": n}

    keys, _, _, _ = ops.interval_events(gi._g_start, gi._g_stop, size=genome.size)
    ms = median_ms(lambda: torch.sort(keys), args.iters)
    out["sort"] = bound(ms, 2 * keys.numel() * 8 * 2)                       # one read and one write, at the least
    sk = torch.sort(keys).values
    ms = median_ms(lambda: ops.pileup_runs(sk, genome.size), args.iters)
    n_runs = int(ops.pileup_runs(sk, genome.size)[2][0])
    out["pileup_runs"] = bound(ms, sk.numel() * 8 + n_runs * 16)
    out["n_runs"] = n_runs
    for name, fn in (("get_pileup_ms", gi.get_pileup), ("get_mask_ms", gi.get_mask), ("merged_ms", gi.merged)):
        out[name] = round(median_ms(fn, args.iters), 4)

    track = gi.get_pileup()
    pchroms, pstart, pstop = synthetic(sizes, args.peaks, 3)
    pstop = pstart + 100
    peaks = genome.get_intervals(bnp.Interval(pchroms, pstart, pstop))
    out["peaks"] = len(peaks)
    out["fused_max_ms"] = round(median_ms(lambda: track[peaks].max(axis=-1), args.iters), 4)
    out["extract_ms"] = round(median_ms(lambda: track[peaks]._data, args.iters), 4)

    c_chroms, c_start, c_stop = synthetic(sizes, 100_000, 4)
    _, gs, ge = po.genome_intervals(sizes, c_chroms, c_start, c_stop)
    t0 = time.perf_counter()
    po.event_runs(gs, ge, genome.size)
    out["oracle_100k_s"] = round(time.perf_counter() - t0, 4)

    if args.check:
        m = min(n, 1_000_000)
        sub = gi[torch.arange(m, device=gi._g_start.device)]
        gs, ge = sub._g_start.cpu().numpy(), sub._g_stop.cpu().numpy()
        s, e, v = po.event_runs(gs, ge, genome.size)
        t = sub.get_pileup()._global
        assert t.starts.cpu().numpy().tolist() == s.tolist() and t.values.cpu().numpy().tolist() == v.tolist()
        ps, pe = peaks._g_start[:10_000].cpu().numpy(), peaks._g_stop[:10_000].cpu().numpy()
        want = po.reduce_runs(s, e, v, ps, pe, "max")
        got = sub.get_pileup()[peaks[torch.arange(10_000, device=gi._g_start.device)]].max(axis=-1)
        assert got.cpu().numpy().tolist() == want.tolist()
        out["check"] = "ok"
    print(json.dumps(out))


if __name__ == "__main__":
    main()
