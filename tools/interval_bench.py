"""BED parsing and interval sequences on the device: kernel times against their HBM bound, the end-to-end calls, the
host list path and the NumPy oracle.

    python tools/interval_bench.py [--lines 10000000] [--intervals 1000000] [--iters 20] [--check]

Workload 1: a synthetic 10 M-line BED (chromosome, start, stop; tests/interval_oracle.synthetic_bed) on the device:
bnpk_delimited_columns alone (CUDA-event median over the lines of bnpk_line_split) and BedBuffer.from_raw_buffer end to
end.  Workload 2: 1 M x 100 bp intervals on sacCer3: the interval copy kernel alone and get_interval_sequences end to end
from device intervals; the list path (host ints) on 10 k intervals; the whole of chrIV (the longest contig, 1.5 Mbases)
as fa["chrIV"], wall time around a synchronise; the oracle on one core.  Prints one JSON line with
the card's name and power limit (read-only nvidia-smi query in the same run); --check compares the outputs with the
oracle and the generator's truth."""
import argparse
import gzip
import json
import os
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
from bionumpy_b200.io import BedBuffer  # noqa: E402

from motif_bench import card, median_ms, HBM_BYTES_PER_S  # noqa: E402

import interval_oracle as io_  # noqa: E402

NAMES = ["chr%d" % i for i in range(1, 23)] + ["chrX", "chrY", "chrM"]


def wall_s(fn, iters=3):
    fn()
    torch.cuda.synchronize()
    times = []
    for _ in range(iters):
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        times.append(time.perf_counter() - t0)
    return float(np.median(times))


def bound(ms, n_bytes):
    b = n_bytes / HBM_BYTES_PER_S * 1e3
    return {"kernel_ms": round(ms, 4), "bytes": int(n_bytes), "bound_ms": round(b, 4), "share_of_bound": round(b / ms, 3)}


def parse_case(n_lines, iters, check):
    text, ci, start, stop = io_.synthetic_bed(n_lines, NAMES, seed=5)
    chunk = torch.frombuffer(bytearray(text), dtype=torch.uint8).cuda()
    starts, lens, _ = ops.line_split(chunk, 1, 0, 0, ord("#"), False, 0, max_rows=n_lines)
    kinds = BedBuffer._kinds
    t_kernel = median_ms(lambda: ops.delimited_columns(chunk, starts, lens, kinds), iters)
    # read: the chunk and the line arrays (12 B/line); written: text view (12 B/line) and two int64 columns
    out = {"lines": n_lines, "bytes": len(text), "columns": bound(t_kernel, len(text) + 12 * n_lines + 28 * n_lines)}
    t_line = median_ms(lambda: ops.line_split(chunk, 1, 0, 0, ord("#"), False, 0, max_rows=n_lines), iters)
    out["line_split"] = bound(t_line, len(text) + 12 * n_lines)
    out["from_raw_buffer_ms"] = round(wall_s(lambda: BedBuffer.from_raw_buffer(chunk)) * 1e3, 3)
    if check:
        d = BedBuffer.from_raw_buffer(chunk).get_data()
        ok = np.array_equal(d.start.cpu().numpy(), start) and np.array_equal(d.stop.cpu().numpy(), stop) and \
            np.array_equal(d.chromosome.lengths.cpu().numpy(), np.array([len(n) for n in NAMES])[ci])
        cut = int(np.flatnonzero(np.frombuffer(text[:1 << 22], dtype=np.uint8) == 10)[99_999]) + 1
        t0 = time.perf_counter()
        _, (c2, s2, e2) = io_.parse_delimited(text[:cut], io_.BED)
        out["cpu_oracle_100k_lines_s"] = round(time.perf_counter() - t0, 4)
        ok = ok and s2.tolist() == start[:100_000].tolist() and e2.tolist() == stop[:100_000].tolist() and \
            c2 == [NAMES[i].encode() for i in ci[:100_000]]
        out["identical"] = bool(ok)
    return out


def gather_case(n, iters, check):
    raw = gzip.open(os.path.join(ROOT, "tests", "golden", "sacCer3.fa.gz")).read()
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "sacCer3.fa")
        with open(path, "wb") as f:
            f.write(raw)
        fa = bnp.open_indexed(path)
    index = fa._index
    names = list(index)
    rng = np.random.default_rng(8)
    ci = rng.integers(0, len(names), n)
    rlen = np.array([index[k]["rlen"] for k in names])[ci]
    starts = (rng.random(n) * (rlen - 100)).astype(np.int64)
    chroms = [names[i] for i in ci]
    iv = bnp.Interval(chroms, starts, starts + 100)
    seqs = fa.get_interval_sequences(iv)
    _, text, name_offsets, contigs = fa._name_table()
    from bionumpy_b200.rows import RowView
    rows = RowView(iv.chromosome)
    ids, _ = ops.name_lookup(rows.base, rows.starts, rows.lens, text, name_offsets)
    row_lens, _ = ops.interval_check(fa._file, iv.start, iv.stop, ids, contigs)
    offsets = ops.row_offsets(row_lens)
    total = 100 * n
    t_copy = median_ms(lambda: ops.interval_copy(fa._file, iv.start, iv.stop, offsets, total, ids, contigs), iters)
    t_lookup = median_ms(lambda: ops.name_lookup(rows.base, rows.starts, rows.lens, text, name_offsets), iters)
    # copy: reads the bases (and up to 2 line ends per row) and 28 B of row and contig data, writes the bases
    out = {"intervals": n, "bp": 100, "copy": bound(t_copy, 2 * total + 28 * n),
           "name_lookup": bound(t_lookup, int(rows.lens.sum().item()) + 16 * n),
           "get_interval_sequences_ms": round(wall_s(lambda: fa.get_interval_sequences(iv)) * 1e3, 3)}
    m = 10_000
    host = list(zip(chroms[:m], starts[:m].tolist(), (starts[:m] + 100).tolist()))
    out["list_path_10k_s"] = round(wall_s(lambda: fa.get_interval_sequences(host), 1), 4)
    out["whole_contig"] = {"name": "chrIV", "bases": index["chrIV"]["rlen"],
                           "ms": round(wall_s(lambda: fa["chrIV"], iters) * 1e3, 3)}
    t0 = time.perf_counter()
    flat, _ = io_.interval_sequences(raw, index, chroms[:m], starts[:m].tolist(), (starts[:m] + 100).tolist())
    out["cpu_oracle_10k_s"] = round(time.perf_counter() - t0, 4)
    if check:
        got = seqs.ravel().raw().cpu().numpy()
        ok = np.array_equal(got[:flat.size], flat) and np.array_equal(seqs.lengths.cpu().numpy(), np.full(n, 100))
        contig = {}
        for k in names:
            i = index[k]
            body = np.frombuffer(raw, dtype=np.uint8)[i["offset"]: i["offset"] + (i["rlen"] // i["lenc"] + 1) * i["lenb"]]
            contig[k] = np.delete(body, np.arange(i["lenc"], body.size, i["lenb"]))[:i["rlen"]]
        whole = np.concatenate([contig[k] for k in names])
        base = np.concatenate([[0], np.cumsum([index[k]["rlen"] for k in names])])[ci]
        want = whole[(base + starts)[:, None] + np.arange(100)].reshape(-1)
        out["identical"] = bool(ok and np.array_equal(got, want) and
                                np.array_equal(fa["chrIV"].raw().cpu().numpy(), contig["chrIV"]))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lines", type=int, default=10_000_000)
    ap.add_argument("--intervals", type=int, default=1_000_000)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--check", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("interval_bench needs a CUDA device")
    name, limit = card()
    result = {"card": name, "power_limit": limit, "parse": parse_case(args.lines, args.iters, args.check)}
    torch.cuda.empty_cache()
    result["gather"] = gather_case(args.intervals, args.iters, args.check)
    print(json.dumps(result))
    if args.check and not (result["parse"]["identical"] and result["gather"]["identical"]):
        raise SystemExit("interval_bench: output differs from the oracle")


if __name__ == "__main__":
    main()
