"""BAM reading on the GPU: kernel times of the record split, the fields and the unpack, their share of the HBM bound,
the split on decoy records, bnp.open(...).read() and read_intervals(...).get_pileup() end to end, and the plain
Python oracle on one core.  Prints one JSON object (and writes it to --out).

The kernel input is a seeded synthetic BAM body of --records records of 150 bases (names of 8..39 bytes, 1-3 cigar
ops, 0-47 aux bytes), built as 100 k distinct records repeated, placed on the device directly from the inflated
bytes; the end-to-end file is a BGZF file of --e2e-records of those records."""
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

import bam_oracle as bo                       # noqa: E402
import bionumpy_b200 as bnp                   # noqa: E402
from bionumpy_b200 import ops                 # noqa: E402

HBM = 3.35e12                                 # H100 SXM data sheet, bytes/s
NAMES = [f"chr{i}" for i in range(1, 23)]
SIZE = 1 << 28


def records(n, seed=0):
    rng = np.random.default_rng(seed)
    out = []
    for i in range(n):
        nc = int(rng.integers(1, 4))
        lens = rng.integers(1, 50, nc - 1).tolist()
        cig = [(0, 150 - sum(lens[::2]))] + [(int(rng.choice([1, 2, 4])), int(x)) for x in lens]
        out.append(bo.record_bytes(ref_id=int(rng.integers(0, len(NAMES))), pos=int(rng.integers(0, SIZE - 1000)),
                                   name=b"r%0*d" % (int(rng.integers(7, 39)), i), mapq=int(rng.integers(0, 61)),
                                   flag=int(rng.integers(0, 2)) * 16, cigar=cig,
                                   seq=rng.integers(1, 16, 150).tolist(), qual=rng.integers(0, 41, 150).tolist(),
                                   aux=bytes(int(rng.integers(0, 48)))))
    return out


def events(fn, reps):
    fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--records", type=int, default=10_000_000)
    ap.add_argument("--e2e-records", type=int, default=1_000_000)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()[0]
    res = {"gpu": gpu}
    base = records(100_000)
    t0 = time.perf_counter()
    names, _, got, _ = bo.parse_bam(bo.header_bytes(NAMES, [SIZE] * len(NAMES)) + b"".join(base))
    res["oracle_100k_records_s"] = time.perf_counter() - t0
    body = b"".join(base) * (args.records // len(base))
    n_rec = len(base) * (args.records // len(base))
    d = torch.frombuffer(bytearray(body), dtype=torch.uint8).cuda()
    del body
    res["inflated_bytes"] = d.numel()
    n_ref = len(NAMES)
    starts, status = ops.bam_split(d, n_ref)
    st = ops.read_status(status)
    assert st.n_records == n_rec and st.n_complete_bytes == d.numel()
    res["walked_again"] = st.n_values
    starts = starts[:n_rec]
    res["split_ms"] = events(lambda: ops.bam_split(d, n_ref), args.reps)
    res["fields_ms"] = events(lambda: ops.bam_fields(d, starts, status), args.reps)
    f = ops.bam_fields(d, starts, status)
    l_seq, n_cig = f[9].to(torch.int32), f[7].to(torch.int32)
    so, co = ops.row_offsets(l_seq), ops.row_offsets(n_cig)
    n_bases, n_ops = int(so[-1]), int(co[-1])
    res["sequence_ms"] = events(lambda: ops.bam_sequence(d, f[8], so, n_bases), args.reps)
    res["cigar_ms"] = events(lambda: ops.bam_cigar(d, f[6], co, n_ops), args.reps)
    # bytes the kernels must move: split reads every record header and writes its start; fields reads the header,
    # the start and the cigar words and writes 12 int64; unpack reads the packed bases / cigar words and writes one
    # byte per base / 9 bytes per op
    need = {"split": n_rec * (36 + 8), "fields": n_rec * (36 + 8 + 96) + 4 * n_ops,
            "sequence": (n_bases + 1) // 2 + n_bases + 16 * n_rec, "cigar": 4 * n_ops + 9 * n_ops + 16 * n_rec}
    for k, v in need.items():
        res[f"{k}_hbm_share"] = v / HBM / (res[f"{k}_ms"] / 1e3)
    del d, starts, f
    torch.cuda.empty_cache()
    # decoys: long records whose aux holds copies of a valid record chain
    chain = b"".join(bo.record_bytes(ref_id=0, name=b"d", seq=[1, 2, 3], qual=b"\x05\x06\x07") for _ in range(3))
    rng = np.random.default_rng(1)
    dec = []
    for i in range(2000):
        dec += base[i * 20:(i + 1) * 20]
        payload = chain * int(rng.integers(100, 1000))
        dec.append(bo.record_bytes(ref_id=1, name=b"decoy", seq=[1] * 10, cigar=[(0, 10)],
                                   aux=b"ZBBC" + len(payload).to_bytes(4, "little") + payload))
    dd = torch.frombuffer(bytearray(b"".join(dec)), dtype=torch.uint8).cuda()
    s2, st2 = ops.bam_split(dd, n_ref)
    st2 = ops.read_status(st2)
    assert st2.n_records == len(dec)
    res["decoy_bytes"], res["decoy_walked_again"] = dd.numel(), st2.n_values
    res["decoy_split_ms"] = events(lambda: ops.bam_split(dd, n_ref), args.reps)
    del dd, s2
    # end to end
    with tempfile.TemporaryDirectory() as tmp:
        path, sizes = os.path.join(tmp, "e2e.bam"), os.path.join(tmp, "g.sizes")
        e2e = base * max(1, args.e2e_records // len(base))
        bo.write_bam(path, NAMES, [SIZE] * len(NAMES), e2e)
        with open(sizes, "w") as fh:
            fh.writelines(f"{n}\t{SIZE}\n" for n in NAMES)
        res["e2e_records"], res["e2e_file_bytes"] = len(e2e), os.path.getsize(path)
        from bionumpy_b200.io.ingest import _GzipSource

        def inflate():
            src = _GzipSource(path)
            while not src.finish(src.start(64 << 20))[2]:
                pass
        g = bnp.Genome.from_file(sizes)
        for name, fn in (("inflate_s", inflate), ("read_s", lambda: bnp.open(path).read().sequence),
                         ("pileup_s", lambda: g.read_intervals(path).get_pileup())):
            fn()
            torch.cuda.synchronize()
            t = []
            for _ in range(3):
                t0 = time.perf_counter()
                fn()
                torch.cuda.synchronize()
                t.append(time.perf_counter() - t0)
            res[name] = min(t)
        res["read_inflate_share"] = res["inflate_s"] / res["read_s"]
        res["pileup_inflate_share"] = res["inflate_s"] / res["pileup_s"]
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
