"""Writer times on the device and end to end: the format kernel (bnpk_format_records) and bnp.open(path, "w").write.

    python tools/write_bench.py [--reads 10000000] [--iters 20] [--check]

Workload 1: synthetic 150 bp reads (ops.synth_fastq, 317 B per record) resident on the device; the record chunk's
fields are views into that chunk (names and qualities as the FASTQ buffer gives them, sequences as text), written as
FASTQ.  Workload 2: sacCer3 (17 chromosomes) as one chunk, written as FASTA wrapped at 80 bases.  Kernel times are
CUDA-event medians of repeated launches after warm-up; each is set against its bound: the field bytes read + 36 B of
views and 8 B of offsets per entry + the bytes written, at the data-sheet 3.35 TB/s.  End to end: write() of the reads
to a plain file and to a .fq.gz (BGZF, deflated on the ingest thread pool) in a temporary directory, wall time.  The
NumPy writer oracle (tests/write_oracle.py) on one core for 100 k reads.  Prints one JSON line with the card's name and
power limit (read-only nvidia-smi query in the same run); --check compares the formatted chunk with the input bytes."""
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
from bionumpy_b200 import _native as nv, ops  # noqa: E402
from bionumpy_b200.io import ingest, write as bw  # noqa: E402

HBM_BYTES_PER_S = 3.35e12          # H100 SXM data sheet


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    name, limit = (q[torch.cuda.current_device()].split(", ") + ["?"])[:2] if q else ("?", "?")
    return name, limit


def median_ms(fn, iters, warmup=3):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    times = []
    for _ in range(iters):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        times.append(a.elapsed_time(b))
    return float(np.median(times))


def kernel_case(entries, buffer_type, iters):
    fmt, width = buffer_type._write_format()
    fields = bw.entry_fields(entries, fmt)
    f = bw.Formatted(fields, fmt, width)
    out = torch.empty(f.size, dtype=torch.uint8, device=f.offsets.device)
    ms = median_ms(lambda: f.slice(0, f.size, out), iters)
    n = fields[1][2].numel()
    field_bytes = sum(int(x[2].to(torch.int64).sum().item()) for x in fields if x is not None)
    bound_bytes = field_bytes + 36 * n + 8 * n + f.size
    return {"entries": n, "bytes_written": f.size, "kernel_ms": round(ms, 4),
            "bound_ms": round(bound_bytes / HBM_BYTES_PER_S * 1e3, 4),
            "fraction_of_bound": round(bound_bytes / HBM_BYTES_PER_S * 1e3 / ms, 3),
            "offsets_ms": round(median_ms(lambda: ops.format_offsets(fmt, width, fields), max(iters // 2, 3)), 4)}, out


def end_to_end(entries, path, reps=3):
    times = []
    for _ in range(reps):
        torch.cuda.synchronize()
        t = time.perf_counter()
        with bnp.open(path, "w") as f:
            f.write(entries)
        times.append(time.perf_counter() - t)
    size = os.path.getsize(path)
    return {"seconds": round(float(np.median(times)), 4), "file_bytes": size}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reads", type=int, default=10_000_000)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--check", action="store_true")
    a = ap.parse_args()
    torch.cuda.set_device(0)
    name, limit = card()
    res = {"tool": "write_bench", "gpu": name, "power_limit": limit, "reads": a.reads}

    chunk = ops.synth_fastq(a.reads, device="cuda")
    entries = bnp.FastQBuffer.from_raw_buffer(chunk).get_data()
    res["fastq_150bp"], text = kernel_case(entries, bnp.FastQBuffer, a.iters)
    if a.check:
        res["check_fastq_bytes_equal"] = bool(torch.equal(text, chunk))
    del text

    with gzip.open(os.path.join(ROOT, "tests", "golden", "sacCer3.fa.gz")) as f:
        genome = f.read()
    sac = bnp.MultiLineFastaBuffer.from_raw_buffer(np.frombuffer(genome + b">", dtype=np.uint8)).get_data()
    old = bnp.MultiLineFastaBuffer.n_characters_per_line
    bnp.MultiLineFastaBuffer.n_characters_per_line = 80
    res["saccer3_width80"], _ = kernel_case(sac, bnp.MultiLineFastaBuffer, a.iters)
    if a.check:
        bnp.MultiLineFastaBuffer.n_characters_per_line = 50
        res["check_saccer3_width50_equal"] = bytes(bnp.MultiLineFastaBuffer.from_data(sac).raw().cpu().numpy()) == genome
    bnp.MultiLineFastaBuffer.n_characters_per_line = old

    with tempfile.TemporaryDirectory() as tmp:
        res["write_plain_fq"] = end_to_end(entries, os.path.join(tmp, "out.fq"))
        res["write_bgzf_fq_gz"] = end_to_end(entries, os.path.join(tmp, "out.fq.gz"), reps=1)
        res["write_bgzf_fq_gz"]["deflate_threads"] = ingest._pool()._max_workers
        res["write_plain_fq"]["GB_per_s"] = round(chunk.numel() / res["write_plain_fq"]["seconds"] / 1e9, 2)
        res["write_bgzf_fq_gz"]["GB_per_s"] = round(chunk.numel() / res["write_bgzf_fq_gz"]["seconds"] / 1e9, 3)
        if a.check:
            with open(os.path.join(tmp, "out.fq"), "rb") as f:
                head = f.read(1 << 20)
            res["check_file_head_equal"] = head == bytes(chunk[:len(head)].cpu().numpy())

    import write_oracle as wo
    from oracle import bnp_oracle as oracle
    host = oracle.synthetic_fastq(0, 100_000)
    fields = wo.read_fastq(host)
    t = time.perf_counter()
    cpu = wo.fastq_text(*fields)
    res["numpy_oracle_100k_reads_s"] = round(time.perf_counter() - t, 4)
    if a.check:
        res["check_oracle_equal"] = bool(np.array_equal(cpu, host))
    print(json.dumps(res))


if __name__ == "__main__":
    main()
