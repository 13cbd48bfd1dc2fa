"""String and pattern match kernel times (K8) on the device: materialised matches and the fused per-row count.

    python tools/match_bench.py [--reads 10000000] [--iters 20] [--check]

Workload 1: synthetic 150 bp reads (ops.synth_fastq), the sequence field of the device-resident chunk, on both routes:
raw text (the byte-LUT kernel, as ``match_string(chunk.sequence, "ACT")`` runs it) and DNAEncoding (the 2-bit kernel),
with "ACT", the 13-bp adapter AGATCGGAAGAGC, "[AG].[AT]" and "AA.{,1}[CT]".  Workload 2: the whole of sacCer3 (17
chromosome rows, cut into pieces as the matchers do) with "CG" and a 30-column pattern.  Times are CUDA-event medians of
repeated launches after warm-up.  Prints one JSON line with the card's name and power limit (read-only nvidia-smi query
in the same run), the algorithmic bytes of every case (sequence bytes + 12 B per row, + 1 B per position materialised
or 8 B per row fused) and each kernel's share of the data-sheet HBM bound, and with --check an oracle check of a subset
and the single-core time of a NumPy restatement (sliding windows compared with the pattern) on 100 k reads."""
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
from bionumpy_b200.encoded_array import BaseEncoding, EncodedArray, EncodedRaggedArray  # noqa: E402
from bionumpy_b200.sequence.string_matcher import FixedLenRegexMatcher, RegexMatcher, StringMatcher  # noqa: E402

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


def case(name, seq, matcher, mode, iters):
    """Times of the materialised matches and the fused count on pre-split rows (the kernels alone: offsets, sets and
    status made once)."""
    pat = matcher._pattern
    rows = pat.rows(seq)
    same = mode == "same"
    offsets = ops.row_offsets(rows.lens, 0 if same else pat.span - 1)
    groups, p_off, total, _ = pat._pieces(rows, same, offsets)
    total = int(offsets[-1].item()) if total is None else total
    out = torch.empty(total, dtype=torch.uint8, device=rows.base.device)
    status = nv.new_status(rows.base.device)
    launch = pat._launch_args(rows)
    prepared = [(g, s, p_off if idx is None else p_off[torch.cat([idx, idx[-1:] + 1])]) for g, s, idx in groups]

    def run_matches():
        for g, s, off in prepared:
            ops.rows_match(g.base, g.starts, g.lens, *launch, same=s, lut=rows.lut, offsets=off, status=status, out=out)

    def run_count():
        for g, s, _ in prepared:
            ops.rows_match_count(g.base, g.starts, g.lens, *launch, same=s, lut=rows.lut, status=status)

    t_m, t_c = median_ms(run_matches, iters), median_ms(run_count, iters)
    n_bases = int(rows.lens.to(torch.int64).sum().item())
    n_rows = sum(int(g.lens.numel()) for g, _, _ in groups)
    read = n_bases + 12 * n_rows
    res = {}
    for kind, t, written in (("matches", t_m, total), ("count", t_c, 8 * n_rows)):
        bound = (read + written) / HBM_BYTES_PER_S * 1e3
        res[kind] = {"kernel_ms": round(t, 4), "bytes": read + written, "bound_ms": round(bound, 4),
                     "share_of_bound": round(bound / t, 3)}
    return {"case": name, "route": "2-bit" if pat.alphabet_size == 4 else "byte-LUT", "span": pat.span,
            "sub_patterns": len(pat.sub_lens), "rows": n_rows, "bases": n_bases, "positions": total, **res}


def numpy_restatement(seqs, pattern):
    """The matches of a literal pattern in rows of equal length, as sliding windows compared with the pattern."""
    windows = np.lib.stride_tricks.sliding_window_view(seqs, len(pattern), axis=1)
    return np.all(windows == np.frombuffer(pattern.encode(), dtype=np.uint8), axis=-1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reads", type=int, default=10_000_000)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--check", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("match_bench needs a CUDA device")
    name, limit = card()
    result = {"card": name, "power_limit": limit, "cases": []}

    chunk = ops.synth_fastq(args.reads)
    starts, lens, _ = ops.line_split(chunk, 4, 1)
    seq = EncodedRaggedArray(EncodedArray(chunk, BaseEncoding), lens, starts=starts)
    for matcher, mode, tag in (
            (StringMatcher("ACT", BaseEncoding), "valid", "reads_ACT_raw"),
            (StringMatcher("ACT", bnp.DNAEncoding), "valid", "reads_ACT_dna"),
            (StringMatcher("AGATCGGAAGAGC", BaseEncoding), "valid", "reads_adapter_raw"),
            (StringMatcher("AGATCGGAAGAGC", bnp.DNAEncoding), "valid", "reads_adapter_dna"),
            (FixedLenRegexMatcher("[AG].[AT]", BaseEncoding), "valid", "reads_[AG].[AT]_raw"),
            (FixedLenRegexMatcher("[AG].[AT]", bnp.DNAEncoding), "valid", "reads_[AG].[AT]_dna"),
            (RegexMatcher("AA.{,1}[CT]", BaseEncoding), "same", "reads_AA.{,1}[CT]_raw"),
            (RegexMatcher("AA.{,1}[CT]", bnp.DNAEncoding), "same", "reads_AA.{,1}[CT]_dna")):
        result["cases"].append(case(tag, seq, matcher, mode, args.iters))
    if args.check:
        import match_oracle as mo
        from oracle import bnp_oracle as o
        n = 2000
        host = chunk[:n * 317].cpu().numpy()
        rows = [host[s:s + L].tobytes() for s, L in zip(starts[:n].cpu().tolist(), lens[:n].cpu().tolist())]
        sub = seq[:n]
        ok = True
        for pattern, alphabet, matcher in (("ACT", None, StringMatcher("ACT", BaseEncoding)),
                                           ("ACT", "ACGT", StringMatcher("ACT", bnp.DNAEncoding)),
                                           ("AA.{,1}[CT]", "ACGT", RegexMatcher("AA.{,1}[CT]", bnp.DNAEncoding))):
            mode = "same" if "{" in pattern else "valid"
            want = mo.matches(rows, pattern, mode, literal=pattern == "ACT", alphabet=alphabet)
            got = matcher.rolling_window(sub, mode=mode)
            ok &= got.sum(axis=-1).cpu().tolist() == [sum(w) for w in want] and got.tolist() == want
        result["oracle_check"] = {"reads": n, "identical": bool(ok)}
        big = o.synthetic_fastq(0, 100_000)
        reads = big.reshape(-1, 317)[:, 13:163]
        t0 = time.perf_counter()
        numpy_restatement(reads, "ACT").sum(axis=1)
        result["numpy_restatement_100k_reads_s"] = round(time.perf_counter() - t0, 4)
    del chunk, starts, lens, seq
    torch.cuda.empty_cache()

    raw = gzip.open(os.path.join(ROOT, "tests", "golden", "sacCer3.fa.gz")).read()
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "sacCer3.fa")
        with open(path, "wb") as f:
            f.write(raw)
        genome = bnp.open(path).read().sequence
        p30 = "CG" + "[AT]" * 4 + "ACGTACGTAC" + "." * 4 + "GGCCAATTGGCCAA"[:10]
        for matcher, tag in ((StringMatcher("CG", BaseEncoding), "sacCer3_CG_raw"),
                             (StringMatcher("CG", bnp.DNAEncoding), "sacCer3_CG_dna"),
                             (FixedLenRegexMatcher(p30, bnp.DNAEncoding), "sacCer3_m30_dna")):
            result["cases"].append(case(tag, genome, matcher, "valid", args.iters))
    print(json.dumps(result))


if __name__ == "__main__":
    main()
