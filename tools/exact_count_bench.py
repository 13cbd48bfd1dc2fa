"""Measure the exact k-mer count (count_kmers_exact / bnpk_rows_kmer_table_insert) and print one JSON line.

Workloads, generated in the run from fixed seeds:
  genome  2 M x 150 bp FASTQ reads drawn at random positions inside the chromosomes of tests/golden/sacCer3.fa.gz
          (each k-mer seen many times), k = 21 and 31, forward and canonical;
  synth   1 M reads of ops.synth_fastq at k = 31 (random reads: nearly every k-mer distinct, the largest table).
For each: the insert kernel alone (CUDA events around single launches into a cleared, pre-sized table), count_kmers_exact
end to end with a capacity= that fits and without one (growth included), distinct k-mers, k-mers/s and table bytes; as
reference points on the same rows the row-driven hashed count into 2^24 buckets (one global atomic per k-mer, same row
walk), count_kmers_hashed(seq, k, 2^24) through the API, and the single-core host np.unique of the oracle's hashes of a
200 k-read subset.  --check compares the subset's exact counts with that np.unique table.

    python tools/exact_count_bench.py [--check] [--reads 2000000] [--synth-reads 1000000] [--out result.json]
"""
import argparse
import gzip
import json
import os
import statistics
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

READ_LEN = 150
B_HASHED = 1 << 24


def parse_args():
    p = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    p.add_argument("--reads", type=int, default=2_000_000, help="genome-sampled reads")
    p.add_argument("--synth-reads", type=int, default=1_000_000, help="ops.synth_fastq reads (0: skip)")
    p.add_argument("--subset", type=int, default=200_000, help="reads of the host np.unique reference / --check")
    p.add_argument("--repeats", type=int, default=5, help="timed repetitions per measurement")
    p.add_argument("--seed", type=int, default=20261015)
    p.add_argument("--check", action="store_true", help="compare the subset's exact counts with the oracle")
    p.add_argument("--out", default=None, help="also write the JSON line to this file")
    return p.parse_args()


def chromosomes():
    text = gzip.open(os.path.join(ROOT, "tests", "golden", "sacCer3.fa.gz")).read().decode()
    chroms = []
    for entry in text.split(">")[1:]:
        seq = "".join(entry.split("\n")[1:])
        chroms.append(np.frombuffer(seq.encode(), dtype=np.uint8))
    return chroms


def genome_fastq(n_reads, seed):
    """FASTQ text of n_reads reads of READ_LEN bases at seeded uniform positions of sacCer3: '@r' + seq + '+' + 'I's."""
    chroms = chromosomes()
    rng = np.random.default_rng(seed)
    starts_per = np.array([c.size - READ_LEN + 1 for c in chroms], dtype=np.int64)
    genome = np.concatenate(chroms)
    offs = np.concatenate([[0], np.cumsum([c.size for c in chroms])[:-1]])
    which = rng.choice(len(chroms), size=n_reads, p=starts_per / starts_per.sum())
    pos = offs[which] + (rng.random(n_reads) * starts_per[which]).astype(np.int64)
    rec = 3 + READ_LEN + 3 + READ_LEN + 1
    out = np.empty((n_reads, rec), dtype=np.uint8)
    out[:, 0:3] = np.frombuffer(b"@r\n", dtype=np.uint8)
    out[:, 3 + READ_LEN:6 + READ_LEN] = np.frombuffer(b"\n+\n", dtype=np.uint8)
    out[:, 6 + READ_LEN:rec - 1] = ord("I")
    out[:, rec - 1] = ord("\n")
    step = 100_000
    cols = np.arange(READ_LEN)
    for i in range(0, n_reads, step):
        out[i:i + step, 3:3 + READ_LEN] = genome[pos[i:i + step, None] + cols]
    return out.reshape(-1)


def event_ms(fn, reps, before=None):
    """Median and min of CUDA-event times of fn(); before() runs outside the timed window."""
    import torch
    ts = []
    for _ in range(reps + 1):
        if before is not None:
            before()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    ts = ts[1:]                                               # the first run is warm-up
    return round(statistics.median(ts), 3), round(min(ts), 3)


def wall_ms(fn, reps):
    import torch
    ts = []
    for _ in range(reps + 1):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        ts.append((time.perf_counter() - t0) * 1e3)
    ts = ts[1:]
    return round(statistics.median(ts), 2), round(min(ts), 2)


def measure(seq, k, canonical, reps):
    import torch
    import bionumpy_b200 as bnp
    from bionumpy_b200 import ops
    from bionumpy_b200.sequence import exact_counts as ec
    from bionumpy_b200.sequence.dna import complement_xor_of
    from bionumpy_b200.sequence.kmers import _source_of, _split_long_rows
    src = _source_of(seq)
    starts, lens, _ = _split_long_rows(src.starts, src.lens, k)
    positions = int(ops.row_offsets(lens, k - 1)[-1].item())
    first = bnp.count_kmers_exact(seq, k, canonical=canonical)
    distinct = len(first)
    assert int(first.counts.sum().item()) == positions
    del first
    slots = ec.slots_for(distinct)
    keys = torch.empty(slots, dtype=torch.int64, device="cuda")
    counts = torch.empty_like(keys)
    n_used = torch.empty(1, dtype=torch.int64, device="cuda")
    cx = complement_xor_of(src.alphabet_encoding) if canonical else 0

    def clear():
        keys.fill_(-1)
        counts.zero_()
        n_used.zero_()

    insert = lambda: ops.rows_kmer_table_insert(src.base, starts, lens, src.enc_mode, k, keys, counts, n_used, cx, src.lut)
    kernel_ms = event_ms(insert, reps, clear)
    assert int(n_used.item()) == distinct
    del keys, counts
    torch.cuda.empty_cache()
    sized_ms = wall_ms(lambda: bnp.count_kmers_exact(seq, k, canonical=canonical, capacity=distinct), reps)
    grown_ms = wall_ms(lambda: bnp.count_kmers_exact(seq, k, canonical=canonical), reps)
    hist = torch.zeros(B_HASHED, dtype=torch.int64, device="cuda")
    if canonical:
        rows_hashed = lambda: ops.rows_kmer_count_canonical(src.base, starts, lens, src.enc_mode, k, cx, B_HASHED, src.lut, hist)
    else:
        rows_hashed = lambda: ops.rows_kmer_count(src.base, starts, lens, src.enc_mode, k, B_HASHED, 0, src.lut, hist)
    hashed_ms = event_ms(rows_hashed, reps)
    api_hashed_ms = wall_ms(lambda: bnp.count_kmers_hashed(seq, k, B_HASHED, canonical=canonical), reps)
    del hist
    torch.cuda.empty_cache()
    return {"k": k, "canonical": canonical, "kmer_positions": positions, "distinct_kmers": distinct,
            "table_slots": slots, "table_bytes": 16 * slots,
            "insert_kernel_ms_median_min": kernel_ms, "insert_Gkmers/s": round(positions / kernel_ms[0] / 1e6, 2),
            "count_kmers_exact_sized_ms_median_min": sized_ms, "count_kmers_exact_grown_ms_median_min": grown_ms,
            "e2e_sized_Gkmers/s": round(positions / sized_ms[0] / 1e6, 2),
            "hashed_rows_2^24_kernel_ms_median_min": hashed_ms,
            "insert_over_hashed": round(kernel_ms[0] / hashed_ms[0], 2),
            "count_kmers_hashed_2^24_api_ms_median_min": api_hashed_ms}


def host_unique(fastq_subset, k, canonical, check_seq=None):
    """Single-core np.unique over the oracle's hashes of the subset; optionally compare count_kmers_exact with it."""
    import bionumpy_b200 as bnp
    from oracle import bnp_oracle as oracle
    _, starts, lens = oracle.fastq_split(fastq_subset)
    flat = oracle.gather_rows(fastq_subset, starts[:, 1], lens[:, 1])
    codes = oracle.encode_flat(flat, oracle.alphabet_lut("ACGT"))
    fn = oracle.canonical_kmers if canonical else oracle.get_kmers
    h = fn(codes, lens[:, 1], k)[0]
    t0 = time.perf_counter()
    u, c = np.unique(h, return_counts=True)
    out = {"reads": int(starts.shape[0]), "kmer_positions": int(h.size), "distinct_kmers": int(u.size),
           "np_unique_ms": round((time.perf_counter() - t0) * 1e3, 1)}
    if check_seq is not None:
        got = bnp.count_kmers_exact(check_seq, k, canonical=canonical)
        same = np.array_equal(got.kmers.cpu().numpy(), u) and np.array_equal(got.counts.cpu().numpy(), c)
        out["check"] = "identical" if same else "DIFFERENT"
    return out


def main():
    args = parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("exact_count_bench needs a CUDA device")
    import bionumpy_b200 as bnp
    from bionumpy_b200 import ops
    from bench import gpu_info
    torch.cuda.set_device(0)
    result = {"metric": "exact_kmer_count", "gpu": gpu_info(0), "read_len": READ_LEN, "hashed_buckets": B_HASHED}

    text = genome_fastq(args.reads, args.seed)
    seq = bnp.FastQBuffer.from_raw_buffer(text).get_data().sequence
    rec = text.size // args.reads
    subset_text = text[:args.subset * rec]
    subset_seq = bnp.FastQBuffer.from_raw_buffer(subset_text).get_data().sequence if args.check else None
    genome = {"reads": args.reads, "runs": []}
    for k in (21, 31):
        for canonical in (False, True):
            run = measure(seq, k, canonical, args.repeats)
            run["host_subset"] = host_unique(subset_text, k, canonical, subset_seq)
            genome["runs"].append(run)
    result["genome_sampled_sacCer3"] = genome
    del seq
    torch.cuda.empty_cache()

    if args.synth_reads:
        chunk = ops.synth_fastq(args.synth_reads)
        sseq = bnp.FastQBuffer.from_raw_buffer(chunk).get_data().sequence
        synth = {"reads": args.synth_reads, "runs": [measure(sseq, 31, False, max(2, args.repeats // 2))]}
        sub = chunk[:args.subset * 317].cpu().numpy()
        synth["runs"][0]["host_subset"] = host_unique(
            sub, 31, False, bnp.FastQBuffer.from_raw_buffer(sub).get_data().sequence if args.check else None)
        result["synth_fastq"] = synth
    line = json.dumps(result)
    print(line, flush=True)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")
    if args.check:
        checks = [r["host_subset"]["check"] for part in ("genome_sampled_sacCer3", "synth_fastq") if part in result
                  for r in result[part]["runs"]]
        if any(c != "identical" for c in checks):
            sys.exit("exact counts differ from the oracle")


if __name__ == "__main__":
    main()
