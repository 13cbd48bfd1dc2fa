"""Time bedGraph reading and float64 tracks on the device and print one JSON line (CUDA-event medians, with the card and
its power limit read by nvidia-smi in the same run), on hg38 with two generated MACS2-shaped tracks (contiguous runs over
every contig, values written as %.5f, about --n lines each):
  from_raw_buffer  BedGraphBuffer.from_raw_buffer of the whole treat file's bytes on the device
  parse            bnpk_parse_float alone over the value column, with the HBM bound: the value bytes, the views
                   (12 bytes a row) and the doubles written (8 bytes a row), at 3.35 TB/s
  get_track        Genome.get_track of the treat rows, end to end
  peak_max / peak_mean
                   the fused per-peak max and mean of --peaks random peaks of 200 to 1000 bases
  ratio            the float combine (treat + 1) / (ctrl + 1)
  read_track       Genome.read_track of the treat file, end to end (host clock)
  numpy_100k       tests/bedgraph_oracle.py reading 100 k lines and filling their dense track on one CPU core.
--check compares the parsed values with the generator's, and on chr21 the track, the ratio and the per-peak max and
mean with dense NumPy."""
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

import bionumpy_b200 as bnp  # noqa: E402
from bionumpy_b200 import ops  # noqa: E402
from bionumpy_b200.io.decimal import pow5_table  # noqa: E402
from bionumpy_b200.io.delimited import BedGraphBuffer  # noqa: E402

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


def digits(x, width):
    """uint8[N, width]: x (int64, >= 0) in decimal, right-aligned, with 0 bytes for the leading zeros (the last digit
    is always kept)."""
    p = 10 ** torch.arange(width - 1, -1, -1, device=x.device, dtype=torch.int64)
    d = (x[:, None] // p) % 10
    keep = torch.cumsum(d != 0, 1) > 0
    keep[:, -1] = True
    return torch.where(keep, d + 48, 0).to(torch.uint8)


def macs_like(sizes, n, rng):
    """(text bytes, per-row chromosome names, starts, stops, values * 1e5 as int64) of contiguous runs over every
    contig, about n rows, generated on the device."""
    total = sum(sizes.values())
    parts, rows = [], []
    for name, size in sizes.items():
        k = max(1, int(round(n * size / total)))
        cuts = torch.sort(torch.randint(1, max(size, 2), (k - 1,), generator=rng, device="cuda")).values
        edges = torch.cat([torch.zeros(1, dtype=torch.int64, device="cuda"), cuts,
                           torch.full((1,), size, dtype=torch.int64, device="cuda")])
        start, stop = edges[:-1], edges[1:]
        value = torch.randint(0, 50_000_000, (k,), generator=rng, device="cuda")
        cols = [torch.tensor(list(name.encode()), dtype=torch.uint8, device="cuda").expand(k, -1),
                torch.full((k, 1), 9, dtype=torch.uint8, device="cuda"), digits(start, 10),
                torch.full((k, 1), 9, dtype=torch.uint8, device="cuda"), digits(stop, 10),
                torch.full((k, 1), 9, dtype=torch.uint8, device="cuda"), digits(value // 100_000, 3),
                torch.full((k, 1), 46, dtype=torch.uint8, device="cuda"),
                (digits(value % 100_000 + 100_000, 6)[:, 1:]),
                torch.full((k, 1), 10, dtype=torch.uint8, device="cuda")]
        m = torch.cat(cols, 1)
        parts.append(m[m != 0])
        rows.append((name, start, stop, value))
    return torch.cat(parts).cpu().numpy().tobytes(), rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--n", type=int, default=20_000_000)
    ap.add_argument("--peaks", type=int, default=1_000_000)
    ap.add_argument("--check", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("track_read_bench needs a CUDA device")
    import bedgraph_oracle as oracle
    genome = bnp.Genome.from_file(os.path.join(ROOT, "tests", "golden", "hg38.chrom.sizes"))
    sizes = genome.get_chromosome_sizes()
    rng = torch.Generator(device="cuda")
    rng.manual_seed(1)
    treat_text, treat_rows = macs_like(sizes, args.n, rng)
    ctrl_text, _ = macs_like(sizes, args.n // 4, rng)
    res = {"card": card(), "lines": sum(int(r[1].numel()) for r in treat_rows), "bytes": len(treat_text)}
    chunk = torch.frombuffer(bytearray(treat_text), dtype=torch.uint8).cuda()
    res["from_raw_buffer_ms"] = median_ms(lambda: BedGraphBuffer.from_raw_buffer(chunk), args.iters)
    buf = BedGraphBuffer.from_raw_buffer(chunk)
    bg = buf.get_data()
    starts, lens, _ = ops.line_split(chunk, 1, 0, 0, ord("#"), False, 0, max_rows=buf.n_lines)
    cols, status = ops.delimited_columns(chunk, starts, lens, BedGraphBuffer._kinds)
    table = pow5_table(chunk.device)
    res["parse_ms"] = median_ms(lambda: ops.parse_float(chunk, cols[3][0], cols[3][1], 3, table, status), args.iters)
    moved = int(cols[3][1].to(torch.int64).sum()) + 20 * buf.n_lines
    res["parse_hbm_fraction"] = moved / HBM / (res["parse_ms"] * 1e-3)
    res["get_track_ms"] = median_ms(lambda: genome.get_track(bg), args.iters)
    treat = genome.get_track(bg)
    ctrl = genome.get_track(BedGraphBuffer.from_raw_buffer(torch.frombuffer(bytearray(ctrl_text),
                                                                            dtype=torch.uint8).cuda()).get_data())
    res["treat_runs"] = int(treat._global.values.numel())
    g = torch.Generator().manual_seed(2)
    names = list(sizes)
    lens_ = torch.tensor([sizes[n] for n in names])
    which = torch.randint(0, len(names), (args.peaks,), generator=g)
    width = torch.randint(200, 1000, (args.peaks,), generator=g)
    pstart = (torch.rand(args.peaks, generator=g) * (lens_[which] - 1000).clamp(min=1)).to(torch.int64)
    peaks = genome.get_intervals(bnp.Interval([names[i] for i in which.tolist()], pstart.numpy(),
                                              (pstart + width).clamp(max=lens_[which]).numpy()))
    res["peak_max_ms"] = median_ms(lambda: treat[peaks].max(axis=-1), args.iters)
    res["peak_mean_ms"] = median_ms(lambda: treat[peaks].mean(axis=-1), args.iters)
    res["ratio_ms"] = median_ms(lambda: (treat + 1) / (ctrl + 1), args.iters)
    with tempfile.TemporaryDirectory() as tmp:
        path = os.path.join(tmp, "treat_pileup.bdg")
        with open(path, "wb") as f:
            f.write(treat_text)
        res["read_track_ms"] = host_ms(lambda: genome.read_track(path), max(args.iters // 5, 1))
        small = os.path.join(tmp, "small.bdg")
        cut = 0
        for _ in range(100_000):
            cut = treat_text.index(b"\n", cut) + 1
        with open(small, "wb") as f:
            f.write(treat_text[:cut])
        t = time.perf_counter()
        rows = oracle.read_bedgraph(small)
        oracle.dense_track(rows, {rows[0][0]: sizes[rows[0][0]]})
        res["numpy_100k_ms"] = (time.perf_counter() - t) * 1e3
    if args.check:
        # the expected doubles divided on the host: NumPy divides, where a CUDA tensor divided by a scalar is multiplied
        # by its reciprocal
        want = np.concatenate([r[3].cpu().numpy() for r in treat_rows]) / 1e5
        checks = {"values": bool(np.array_equal(bg.value.cpu().numpy().view(np.int64), want.view(np.int64)))}
        name = "chr21"
        r = next(r for r in treat_rows if r[0] == name)
        dense = np.repeat(r[3].cpu().numpy() / 1e5, (r[2] - r[1]).cpu().numpy())
        checks["track"] = bool(np.array_equal(np.asarray(treat[name]).view(np.int64), dense.view(np.int64)))
        ratio = (treat + 1) / (ctrl + 1)
        c = np.asarray(ctrl[name])
        checks["ratio"] = bool(np.array_equal(np.asarray(ratio[name]).view(np.int64),
                                              ((dense + 1) / (c + 1)).view(np.int64)))
        on = (which == names.index(name)).nonzero().reshape(-1)
        sel = peaks[on.cuda()]
        mx, mean = treat[sel].max(axis=-1).cpu().numpy(), treat[sel].mean(axis=-1).cpu().numpy()
        ok_max = ok_mean = True
        for i, (a, b) in enumerate(zip(sel.start.cpu().tolist(), sel.stop.cpu().tolist())):
            ok_max &= bool(mx[i] == dense[a:b].max())
            ok_mean &= abs(mean[i] - float(oracle.exact_sum(dense[a:b])) / (b - a)) <= 1e-12 * abs(mean[i])
        checks["peak_max"], checks["peak_mean"] = ok_max, bool(ok_mean)
        res["check"] = all(checks.values())
        res["checks"] = checks
    print(json.dumps(res))


if __name__ == "__main__":
    main()
