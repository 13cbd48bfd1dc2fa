"""Time GTF reading, the attribute kernel, get_exons and spliced transcript sequences on the GPU.

    python tools/annotation_bench.py [--lines 3400000] [--seed 1] [--reps 5] [--check]

A GENCODE-shaped GTF is generated from the seed with NumPy (no Python loop per line): genes of one transcript and
eight exons, every line ~460 bytes with GENCODE's attribute keys, '-' transcripts listing their exons in descending
order.  Times are CUDA-event medians after a warm-up run; the attribute kernel's rate is its attribute bytes over its
time, against 3.35 TB/s (H100 SXM HBM3).  ``--check`` compares exons and transcript sequences of a 100 k-line slice
with tests/annotation_oracle.py and times the oracle on one CPU core.  Prints one JSON line, with the card and its
power limit."""
import argparse
import gzip
import json
import os
import shutil
import statistics
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
from bionumpy_b200 import ops  # noqa: E402
from bionumpy_b200.io import GTFBuffer  # noqa: E402
from bionumpy_b200.rows import RowView  # noqa: E402
from bionumpy_b200.sequence import get_transcript_sequences  # noqa: E402

HBM_BYTES_PER_S = 3.35e12
EXONS, SPAN, EXON_LEN = 8, 400, 40
FILLER = ('gene_type "protein_coding"; gene_name "GENE1"; level 2; transcript_type "protein_coding"; '
          'transcript_name "TX-201"; exon_number {e}; exon_id "ENSE{x}.1"; protein_id "ENSP00000000001.1"; '
          'transcript_support_level "1"; hgnc_id "HGNC:5"; tag "basic"; tag "Ensembl_canonical"; tag "MANE_Select"; '
          'havana_gene "OTTHUMG00000000001.1";')
LINE = 'chr1\tHAVANA\t{f}\t{a}\t{b}\t.\t{s}\t.\tgene_id "ENSG{g}.1"; transcript_id "ENST{t}.1"; ' + FILLER


def _template(feature, width):
    """One line with '#' digit fields of fixed width, padded with spaces to `width` bytes and a newline."""
    d = "#" * 11
    line = LINE.format(f=feature, a="#" * 9, b="#" * 9, s="#", g=d, t=d, e="#", x=d)
    assert len(line) < width
    return np.frombuffer((line + " " * (width - 1 - len(line)) + "\n").encode(), dtype=np.uint8)


def generate(n_lines, seed, width=460):
    """(uint8 text of n_lines lines, per-line feature codes 0 gene / 1 transcript / 2 exon)."""
    rng = np.random.default_rng(seed)
    per_gene = 2 + EXONS
    n_genes = (n_lines + per_gene - 1) // per_gene
    kind = np.tile(np.array([0, 1] + [2] * EXONS, dtype=np.int8), n_genes)[:n_lines]
    gene = np.repeat(np.arange(n_genes), per_gene)[:n_lines]
    exon = np.tile(np.array([0, 0] + list(range(EXONS))), n_genes)[:n_lines]
    minus = rng.random(n_genes) < 0.5
    exon = np.where(minus[gene] & (kind == 2), EXONS - 1 - exon, exon)       # '-' lists its exons descending
    g0 = gene.astype(np.int64) * SPAN
    start = np.where(kind == 2, g0 + exon * (SPAN // EXONS), g0)
    stop = np.where(kind == 2, start + EXON_LEN, g0 + SPAN - (SPAN // EXONS - EXON_LEN))
    templates = [_template(f, width) for f in ("gene", "transcript", "exon")]
    text = np.stack(templates)[kind]                                         # [n_lines, width]
    fields = [(start, 9), (stop, 9), (gene, 11), (gene, 11), (exon + 1, 1), (gene * EXONS + exon, 11)]
    for t in range(3):
        where = np.flatnonzero(templates[t] == ord("#"))
        rows = kind == t
        runs = np.split(where, np.flatnonzero(np.diff(where) > 1) + 1)
        strand_col = [r for r in runs if len(r) == 1][0]
        text[rows, strand_col[0]] = np.where(minus[gene[rows]], ord("-"), ord("+"))
        numbers = iter(fields)
        for r in runs:
            if len(r) == 1 and r[0] == strand_col[0]:
                continue
            values, w = next(numbers)
            assert len(r) == w
            digits = (values[rows, None] // 10 ** np.arange(w - 1, -1, -1)) % 10 + ord("0")
            text[np.ix_(np.flatnonzero(rows), r)] = digits.astype(np.uint8)
    return text.reshape(-1), kind, int(g0[-1] + SPAN)


def timed(fn, reps):
    fn()
    torch.cuda.synchronize()
    times = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        times.append(a.elapsed_time(b) / 1e3)
    return statistics.median(times)


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else torch.cuda.get_device_name()
    except (OSError, subprocess.SubprocessError):
        return torch.cuda.get_device_name()


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--lines", type=int, default=3400000)
    p.add_argument("--seed", type=int, default=1)
    p.add_argument("--reps", type=int, default=5)
    p.add_argument("--check", action="store_true")
    args = p.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("annotation_bench needs a CUDA device")
    host, kind, genome_size = generate(args.lines, args.seed)
    chunk = torch.from_numpy(host).cuda()
    res = {"card": card(), "lines": args.lines, "bytes": int(host.size)}
    res["from_raw_buffer_s"] = timed(lambda: GTFBuffer.from_raw_buffer(chunk), args.reps)
    entries = GTFBuffer.from_raw_buffer(chunk).get_data()
    attr = RowView(entries.atributes)
    attr_bytes = int(attr.lens.to(torch.int64).sum())
    keys = ["gene_id", "transcript_id", "exon_id"]
    t = timed(lambda: ops.attribute_values(attr.base, attr.starts, attr.lens, keys, nv.ATTR_GTF), args.reps)
    res.update(attribute_kernel_s=t, attribute_bytes=attr_bytes, attribute_GBps=attr_bytes / t / 1e9,
               attribute_fraction_of_hbm_bound=attr_bytes / HBM_BYTES_PER_S / t)
    res["get_exons_s"] = timed(lambda: entries.get_exons(), args.reps)
    rng = np.random.default_rng(args.seed + 1)
    genome = bnp.EncodedArray(torch.from_numpy(np.frombuffer(b"ACGT", dtype=np.uint8)[
        rng.integers(0, 4, genome_size)].copy()).cuda(), bnp.BaseEncoding)
    res["transcript_sequences_s"] = timed(lambda: get_transcript_sequences(entries, genome), args.reps)
    res["n_exons"] = len(entries.get_exons())

    with tempfile.TemporaryDirectory() as tmp:
        fa = os.path.join(tmp, "sacCer3.fa")
        with gzip.open(os.path.join(ROOT, "tests", "golden", "sacCer3.fa.gz")) as src, open(fa, "wb") as dst:
            shutil.copyfileobj(src, dst)
        gtf = os.path.join(ROOT, "tests", "golden", "sacCer3.ensGene.gtf.gz")

        def sac():
            ann = bnp.Genome.from_file(fa).read_annotation(gtf)
            introns = ann.transcripts.get_mask() & ~ann.exons.get_mask()
            tx = get_transcript_sequences(bnp.open(gtf).read(), bnp.open_indexed(fa))
            return introns, tx
        sac()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        _, tx = sac()
        torch.cuda.synchronize()
        res["sacCer3_end_to_end_s"] = time.perf_counter() - t0
        res["sacCer3_transcripts"] = len(tx.sequence)

    if args.check:
        import annotation_oracle as ao
        n = min(100000, args.lines)
        n -= n % (2 + EXONS)
        part = host[:n * 460].tobytes()
        t0 = time.perf_counter()
        rows = ao.read(part, False)
        want = ao.select(rows, "exon", False)
        res["oracle_100k_lines_s"] = time.perf_counter() - t0
        got = GTFBuffer.from_raw_buffer(torch.from_numpy(host[:n * 460].copy()).cuda()).get_data()
        exons = got.get_exons()

        def texts(field):
            v = RowView(field)
            b, s, l = v.base.cpu().numpy().tobytes(), v.starts.cpu().tolist(), v.lens.cpu().tolist()
            return [b[i:i + k] for i, k in zip(s, l)]
        ok = all(texts(getattr(exons, k)) == [r[k] for r in want] for k in ("gene_id", "transcript_id", "exon_id"))
        ok &= exons.start.cpu().tolist() == [r["start"] for r in want]
        g = genome.raw().cpu().numpy().tobytes()
        seqs = ao.transcript_sequences(want, lambda c, s, e: g[s:e])
        tx = get_transcript_sequences(got, genome)
        ok &= texts(tx.sequence) == [s for _, s in seqs] and texts(tx.name) == [t for t, _ in seqs]
        res["oracle_agrees"] = bool(ok)
    print(json.dumps(res))
    if args.check and not res["oracle_agrees"]:
        raise SystemExit(1)


if __name__ == "__main__":
    main()
