"""Time the interval-set operations on the device and print one JSON line (CUDA-event medians, with the card and its
power limit read by nvidia-smi in the same run):
  combine_and        bnpk_runs_combine of two hg38 masks, each of 10 M synthetic 150-bp intervals, with its bound
                     (16 B read per input run and 16 B written per output run)
  combine_gt         `pileup > 4` on the pileup of the first set
  intersect / global_intersect of two 5 M-row sets (rows grouped by chromosome), split into the sorts and the kernel
  count_overlap, jaccard end to end, and the oracle on one CPU core for 100 k rows.
--check compares every result with tests/interval_sets_oracle.py."""
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
sys.path.insert(0, os.path.join(ROOT, "tests"))

import bionumpy_b200 as bnp  # noqa: E402
from bionumpy_b200 import _native as nv, ops  # noqa: E402
from bionumpy_b200.arithmetics import count_overlap, global_intersect, intersect, jaccard  # noqa: E402
from bionumpy_b200.arithmetics.intervals import chromosome_ranks, lexsort_order  # noqa: E402


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


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip().splitlines()
    return out[0] if out else "unknown"


def synthetic(genome, n, rng):
    names = list(genome.chrom_sizes)
    sizes = np.array([genome.chrom_sizes[c] for c in names])
    c = np.sort(rng.choice(len(names), n, p=sizes / sizes.sum()))      # grouped by chromosome, as BED files are
    s = (rng.random(n) * (sizes[c] - 150)).astype(np.int64)
    return bnp.Interval([names[i] for i in c], s, s + 150), ([names[i] for i in c], s, s + 150)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--check", action="store_true")
    args = ap.parse_args()
    rng = np.random.default_rng(0)
    genome = bnp.Genome.from_file(os.path.join(ROOT, "tests", "golden", "hg38.chrom.sizes"))
    out = {"card": card()}
    ia, ha = synthetic(genome, 10_000_000, rng)
    ib, hb = synthetic(genome, 10_000_000, rng)
    ga, gb = genome.get_intervals(ia), genome.get_intervals(ib)
    ma, mb = ga.get_mask(), gb.get_mask()
    pile = ga.get_pileup()
    for name, x, y, op in (("combine_and", ma._global, mb._global, nv.OP_AND),
                           ("combine_gt", pile._global, None, nv.OP_GT)):
        if y is None:
            ys = torch.arange(2, dtype=torch.int64, device="cuda") * genome.size
            yv = torch.full((1,), 4, dtype=torch.int64, device="cuda")
        else:
            ys, yv = y._events, y._values64()
        xv = x._values64()
        ms = median_ms(lambda: ops.runs_combine(x._events, xv, ys, yv, op), args.iters)
        n_out = int(ops.runs_combine(x._events, xv, ys, yv, op)[2][0])
        n_in = xv.numel() + yv.numel()
        out[name] = {"ms": round(ms, 4), "runs_in": n_in, "runs_out": n_out,
                     "GBps": round((16 * n_in + 16 * n_out) / ms / 1e6, 1)}
    sa, sb = ia[torch.arange(5_000_000, device="cuda")], ib[torch.arange(5_000_000, device="cuda")]
    start = torch.cat([sa.start, sb.start])
    stop = torch.cat([sa.stop, sb.stop])
    t_sort = median_ms(lambda: (torch.sort(start, stable=True), torch.sort(stop)), args.iters)
    order = torch.sort(start, stable=True).indices
    ss, es = start[order], torch.sort(stop).values
    t_kernel = median_ms(lambda: ops.interval_intersect(ss, es), args.iters)
    t_all = median_ms(lambda: intersect(sa, sb), max(args.iters // 4, 3))
    out["intersect"] = {"ms": round(t_all, 3), "sort_ms": round(t_sort, 3), "kernel_ms": round(t_kernel, 4),
                        "kernel_GBps": round(17 * ss.numel() / t_kernel / 1e6, 1)}
    ra, rb = chromosome_ranks([sa.chromosome, sb.chromosome])
    rank = torch.cat([ra, rb])
    t_gsort = median_ms(lambda: (lexsort_order(start, rank), lexsort_order(stop, rank)), args.iters)
    t_gall = median_ms(lambda: global_intersect(sb, sa), max(args.iters // 4, 3))
    out["global_intersect"] = {"ms": round(t_gall, 3), "sort_ms": round(t_gsort, 3)}
    out["count_overlap_ms"] = round(median_ms(lambda: count_overlap(sa, sb), args.iters), 3)
    out["jaccard_ms"] = round(median_ms(lambda: jaccard(genome, ia, ib), max(args.iters // 4, 3)), 2)
    import interval_sets_oracle as so
    small_a = (ha[0][:100_000], ha[1][:100_000], ha[2][:100_000])
    small_b = (hb[0][:100_000], hb[1][:100_000], hb[2][:100_000])
    t0 = time.perf_counter()
    so.intersect(small_a, small_b)
    so.count_overlap(small_a, small_b)
    out["oracle_100k_intersect_and_count_ms"] = round(1000 * (time.perf_counter() - t0), 1)
    if args.check:
        hsa = (ha[0][:5_000_000], ha[1][:5_000_000], ha[2][:5_000_000])
        hsb = (hb[0][:5_000_000], hb[1][:5_000_000], hb[2][:5_000_000])
        rows, stops = so.intersect(hsa, hsb)
        got = intersect(sa, sb)
        starts = np.concatenate([hsa[1], hsb[1]])
        ok = got.start.cpu().numpy().tolist() == starts[rows].tolist() and got.stop.cpu().numpy().tolist() == stops.tolist()
        ok &= count_overlap(sa, sb) == so.count_overlap(hsa, hsb)
        sizes = genome.chrom_sizes
        ok &= jaccard(genome, ia, ib) == so.jaccard(sizes, ha, hb)
        both = (ma & mb).sum().item()
        ((x, _), _) = so.contingency_table(ha, hb, genome.size)
        ok &= both == x
        out["check"] = bool(ok)
        if not ok:
            print(json.dumps(out))
            sys.exit(1)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
