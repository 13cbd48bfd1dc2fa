"""A/B timing of the fused k-mer count between two builds of libbnpk.so, alternating on one card.

    python tools/ws_ab_bench.py BASE_LIB NEW_LIB [--rounds 7] [--launches 20] [--reads 10000000] [--out DIR]

Times `ops.chunk_kmer_count` at the shape bench.py measures (10 M x 150 bp synthetic reads, k = 31, 2^14 bins), with
CUDA events around every launch.  Each round runs a few warm-up launches and then `launches` timed launches of one
library, then the same for the other; the order alternates from round to round.  The histogram and the status words of
the two builds must be identical.  Prints the card's name and power limit, each round's median per library, and one
JSON line (also written to DIR/ws_ab.json with --out)."""
import argparse
import json
import os
import statistics
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from bionumpy_b200 import ops, _native as nv  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader",
                        "-i", str(torch.cuda.current_device())], capture_output=True, text=True)
    return q.stdout.strip() or torch.cuda.get_device_name()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("base_lib")
    ap.add_argument("new_lib")
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--launches", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--reads", type=int, default=10_000_000)
    ap.add_argument("--k", type=int, default=31)
    ap.add_argument("--bins", type=int, default=1 << 14)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()

    libs = {"base": nv.load_library(args.base_lib), "new": nv.load_library(args.new_lib)}
    dev = torch.device("cuda", torch.cuda.current_device())
    chunk = ops.synth_fastq(args.reads, device=dev)

    def use(name):
        nv._lib = libs[name]                      # ops calls go to this build from here on

    # the two builds must compute the same thing at this shape
    outputs = {}
    for name in libs:
        use(name)
        hist, status = ops.chunk_kmer_count(chunk, args.k, args.bins)
        outputs[name] = (hist.cpu(), status.cpu())
    identical = torch.equal(outputs["base"][0], outputs["new"][0]) and torch.equal(outputs["base"][1], outputs["new"][1])

    hist = torch.zeros(args.bins, dtype=torch.int64, device=dev)
    status = nv.new_status(dev)
    medians = {name: [] for name in libs}
    for r in range(args.rounds):
        order = ("base", "new") if r % 2 == 0 else ("new", "base")
        for name in order:
            use(name)
            for _ in range(args.warmup):
                ops.chunk_kmer_count(chunk, args.k, args.bins, hist=hist, status=status)
            ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(args.launches)]
            for a, b in ev:
                a.record()
                ops.chunk_kmer_count(chunk, args.k, args.bins, hist=hist, status=status)
                b.record()
            torch.cuda.synchronize()
            medians[name].append(statistics.median(a.elapsed_time(b) for a, b in ev))
        print(f"round {r}: base {medians['base'][-1]:.4f} ms  new {medians['new'][-1]:.4f} ms", flush=True)

    mb, mn = statistics.median(medians["base"]), statistics.median(medians["new"])
    line = {
        "card": card(),
        "shape": {"reads": args.reads, "k": args.k, "bins": args.bins, "chunk_bytes": chunk.numel()},
        "rounds": args.rounds, "launches_per_round": args.launches,
        "base_round_medians_ms": [round(x, 4) for x in medians["base"]],
        "new_round_medians_ms": [round(x, 4) for x in medians["new"]],
        "base_median_ms": round(mb, 4), "new_median_ms": round(mn, 4),
        "change": round(mn / mb - 1.0, 4),
        "every_new_round_below_every_base_round": max(medians["new"]) < min(medians["base"]),
        "outputs_identical": identical,
    }
    print(json.dumps(line), flush=True)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "ws_ab.json"), "w") as f:
            json.dump(line, f, indent=1)


if __name__ == "__main__":
    main()
