"""Motif-score kernel times (K7) on the device: materialised scores and the fused per-row maximum.

    python tools/motif_bench.py [--reads 10000000] [--iters 20] [--check]

Workload 1: synthetic 150 bp reads (ops.synth_fastq), the sequence field of the device-resident chunk, with MA0080.1
(m = 6) and a random 19-column matrix.  Workload 2: the whole of sacCer3 (17 chromosome rows, cut into pieces as
get_motif_scores does), MA0080.1 and a random 30-column matrix.  Times are CUDA-event medians of repeated launches after
warm-up.  Prints one JSON line with the card's name and power limit (read-only nvidia-smi query in the same run), the
algorithmic bytes and float64 adds of every case, which bound applies, and with --check an oracle check of a subset and
the oracle's single-core time on 100 k reads."""
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
from bionumpy_b200.sequence.kmers import _split_long_rows  # noqa: E402
from bionumpy_b200.sequence.position_weight_matrix import PWM  # noqa: E402

HBM_BYTES_PER_S = 3.35e12          # H100 SXM data sheet
DADD_PER_S = 34e12 / 2             # H100 SXM data sheet FP64 (non-tensor) 34 TFLOP/s counts an FMA as 2


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


def case(name, base, starts, lens, enc_mode, pwm, iters):
    """Times of the scores and the fused max on pre-split rows (the kernels alone: offsets and status made once)."""
    m = pwm.window_size
    mat = pwm.device_matrix(base.device)
    p_starts, p_lens, _ = _split_long_rows(starts, lens, m)
    offsets = ops.row_offsets(p_lens, m - 1)
    total = int(offsets[-1].item())
    scores = torch.empty(total, dtype=torch.float64, device=base.device)
    best = torch.empty(p_lens.numel(), dtype=torch.float64, device=base.device)
    status = nv.new_status(base.device)
    lib = nv.lib()
    args, _ = ops._rows_args(base, p_starts, p_lens)
    st = nv.stream_ptr()

    def run_scores():
        nv.check(lib.bnpk_rows_pwm_scores(*args, enc_mode, None, 4, nv.ptr(mat), m, 0, nv.ptr(offsets),
                                          nv.ptr(scores), nv.ptr(status), st))

    def run_max():
        nv.check(lib.bnpk_rows_pwm_max(*args, enc_mode, None, 4, nv.ptr(mat), m, nv.ptr(best), nv.ptr(status), st))

    t_scores, t_max = median_ms(run_scores, iters), median_ms(run_max, iters)
    n_bases = int(lens.to(torch.int64).sum().item())
    read = n_bases + 12 * p_lens.numel()
    adds = total * m
    out = {}
    for kind, t, written in (("scores", t_scores, 8 * total), ("max", t_max, 8 * p_lens.numel())):
        t_bw, t_fp = (read + written) / HBM_BYTES_PER_S * 1e3, adds / DADD_PER_S * 1e3
        out[kind] = {"kernel_ms": round(t, 4), "bytes": read + written, "dadds": adds,
                     "bound": "memory" if t_bw >= t_fp else "fp64", "bound_ms": round(max(t_bw, t_fp), 4),
                     "share_of_bound": round(max(t_bw, t_fp) / t, 3)}
    del scores
    return {"case": name, "m": m, "rows": int(lens.numel()), "bases": n_bases, "windows": total, **out}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reads", type=int, default=10_000_000)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--check", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("motif_bench needs a CUDA device")
    name, limit = card()
    rng = np.random.default_rng(19)
    ma = bnp.io.read_motif(os.path.join(ROOT, "tests", "golden", "MA0080.1.jaspar"))
    r19, r30 = PWM(rng.normal(size=(4, 19)), "ACGT"), PWM(rng.normal(size=(4, 30)), "ACGT")
    result = {"card": name, "power_limit": limit, "cases": []}

    chunk = ops.synth_fastq(args.reads)
    starts, lens, _ = ops.line_split(chunk, 4, 1)
    for pwm, tag in ((ma, "reads_MA0080.1"), (r19, "reads_m19")):
        result["cases"].append(case(tag, chunk, starts, lens, nv.ENC_ASCII_ACGT, pwm, args.iters))
    if args.check:
        import motif_oracle as mo
        from oracle import bnp_oracle as o
        n = 2000
        host = chunk[:n * 317].cpu().numpy()
        sub_s, sub_l = starts[:n], lens[:n]
        rows = [host[s:s + L] for s, L in zip(sub_s.cpu().tolist(), sub_l.cpu().tolist())]
        codes = o.encode_flat(np.concatenate(rows), o.alphabet_lut("ACGT")).astype(np.int64)
        want, want_lens = mo.motif_scores(codes, sub_l.cpu().numpy(), ma._matrix)
        got, _, _ = ops.rows_pwm_scores(chunk, sub_s, sub_l, nv.ENC_ASCII_ACGT, ma.device_matrix(chunk.device))
        best, _ = ops.rows_pwm_max(chunk, sub_s, sub_l, nv.ENC_ASCII_ACGT, ma.device_matrix(chunk.device))
        ok = np.array_equal(got.cpu().numpy().view(np.int64), want.view(np.int64)) and \
            np.array_equal(best.cpu().numpy().view(np.int64), mo.row_max(want, want_lens).view(np.int64))
        result["oracle_check"] = {"reads": n, "identical": bool(ok)}
        big = o.synthetic_fastq(0, 100_000)
        seq = big.reshape(-1, 317)[:, 13:163].reshape(-1)
        codes = o.encode_flat(seq, o.alphabet_lut("ACGT")).astype(np.int64)
        t0 = time.perf_counter()
        mo.motif_scores(codes, np.full(100_000, 150), ma._matrix)
        result["cpu_oracle_100k_reads_s"] = round(time.perf_counter() - t0, 4)
    del chunk, starts, lens
    torch.cuda.empty_cache()

    raw = gzip.open(os.path.join(ROOT, "tests", "golden", "sacCer3.fa.gz")).read()
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "sacCer3.fa")
        with open(path, "wb") as f:
            f.write(raw)
        seq = bnp.open(path).read().sequence
        base = seq._data.contiguous()
        for pwm, tag in ((ma, "sacCer3_MA0080.1"), (r30, "sacCer3_m30")):
            result["cases"].append(case(tag, base, seq._starts.contiguous(), seq._lens.contiguous(),
                                        nv.ENC_ASCII_ACGT, pwm, args.iters))
    print(json.dumps(result))


if __name__ == "__main__":
    main()
