"""Exact distinct-k-mer counts (count_kmers_exact / KmerCounter / bnpk_rows_kmer_table_insert) against
np.unique(oracle k-mers, return_counts=True), plus the host-side capacity policy and the kernels' build."""
import gzip
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch

from oracle import bnp_oracle as oracle
from helpers import make_fastq

gpu = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def bnp():
    import bionumpy_b200 as bnp
    return bnp


def random_rows(rng, n, max_len, alphabet="ACGT"):
    """Ragged rows with empty and shorter-than-k rows among them."""
    lens = [int(x) for x in rng.integers(0, max_len + 1, size=n)]
    lens[:3] = [0, 1, 2]
    return ["".join(rng.choice(list(alphabet), size=L)) for L in lens]


def oracle_table(strings, k, canonical=False, alphabet="ACGT"):
    flat = np.frombuffer("".join(strings).encode(), dtype=np.uint8)
    codes = oracle.encode_flat(flat, oracle.alphabet_lut(alphabet))
    lens = np.array([len(s) for s in strings], dtype=np.int64)
    h = oracle.canonical_kmers(codes, lens, k, alphabet)[0] if canonical else oracle.get_kmers(codes, lens, k)[0]
    return np.unique(h, return_counts=True)


def assert_table(got, want):
    u, c = want
    assert np.array_equal(got.kmers.cpu().numpy(), u)
    assert np.array_equal(got.counts.cpu().numpy(), c)
    assert len(got) == u.size


# ---------------------------------------------------------------------------------------------------------------
# CPU: capacity policy, argument checks, build
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("seed", range(6))
def test_plan_insert_keeps_the_load_limit_and_covers_every_row_once(seed):
    from bionumpy_b200.sequence import exact_counts as ec
    rng = np.random.default_rng(seed)
    n_rows = int(rng.integers(1, 400))
    pos = rng.integers(0, 300, size=n_rows)
    pos[rng.random(n_rows) < 0.2] = 0                         # rows shorter than k
    if seed % 2:
        pos[rng.integers(0, n_rows)] = 5000                    # one row larger than any batch
    offsets = torch.from_numpy(np.concatenate([[0], np.cumsum(pos)])).to(torch.int64)
    total = int(offsets[-1])
    for first_slots, min_batch, new_frac in ((2, 64, 1.0), (32, 1000, 0.3), (1 << 16, 1 << 20, 1.0), (64, 7, 0.0)):
        slots, n_used, row, done, covered, launches = first_slots, 0, 0, 0, [], 0
        while row < n_rows:
            new_slots, end, end_pos = ec.plan_insert(offsets, row, done, total, n_used, slots, min_batch)
            assert new_slots >= slots and new_slots & (new_slots - 1) == 0
            assert end > row and end_pos == int(offsets[end])
            assert n_used + (end_pos - done) <= ec.MAX_LOAD * new_slots            # the load invariant
            covered.extend(range(row, end))
            n_used += int(round(new_frac * (end_pos - done)))                       # new keys of this launch
            slots, row, done = new_slots, end, end_pos
            launches += 1
        assert covered == list(range(n_rows))
        if n_used + total <= first_slots // 2:
            assert launches == 1


def test_plan_insert_one_launch_when_everything_fits():
    from bionumpy_b200.sequence import exact_counts as ec
    offsets = torch.tensor([0, 10, 10, 25], dtype=torch.int64)
    assert ec.plan_insert(offsets, 0, 0, 25, 0, 64) == (64, 3, 25)
    assert ec.plan_insert(offsets, 0, 0, 25, 7, 64) == (64, 3, 25)
    assert ec.plan_insert(offsets, 1, 10, 25, 17, 64) == (64, 3, 25)
    assert ec.slots_for(16) == 32 and ec.slots_for(17) == 64 and ec.slots_for(1) == 2


def test_plan_insert_grows_and_splits():
    from bionumpy_b200.sequence import exact_counts as ec
    offsets = torch.tensor([0, 10, 20, 30, 40], dtype=torch.int64)
    # 40 positions, 16 slots (limit 8), min batch 20: grow to 64 (limit 32), take rows 0..2 (30 positions)
    assert ec.plan_insert(offsets, 0, 0, 40, 0, 16, min_batch=20) == (64, 3, 30)
    # the free room (limit 32 - 25 used = 7) is below the remaining 10 positions and the min batch: grow to 128
    assert ec.plan_insert(offsets, 3, 30, 40, 25, 64, min_batch=20) == (128, 4, 40)


def test_table_entry_points_reject_bad_arguments():
    from bionumpy_b200 import _native as nv
    lib = nv.load_library()
    null = None
    args = lambda k, cap: (null, 0, null, null, 1, nv.ENC_ASCII_ACGT, null, k, 0, null, null, cap, null, null, null)
    assert lib.bnpk_rows_kmer_table_insert(*args(21, 48)) == nv.E_BADARG
    assert lib.bnpk_rows_kmer_table_insert(*args(21, 0)) == nv.E_BADARG
    assert lib.bnpk_rows_kmer_table_insert(*args(0, 64)) == nv.E_K
    assert lib.bnpk_rows_kmer_table_insert(*args(32, 64)) == nv.E_K
    assert lib.bnpk_kmer_table_rehash(null, null, 64, null, null, 96, null, null, null) == nv.E_BADARG
    assert lib.bnpk_kmer_table_rehash(null, null, 3, null, null, 128, null, null, null) == nv.E_BADARG
    assert nv.ST_TABLE_FULL == 13
    header = open(os.path.join(ROOT, "include", "bnpk.h")).read()
    assert re.search(r"BNPK_ST_TABLE_FULL\s*=\s*13\b", header)


def test_torch_library_registers_the_table_op():
    from bionumpy_b200 import torch_ops
    ops = torch_ops.load()
    assert hasattr(ops, "rows_kmer_table_insert")
    schema = str(torch._C._get_schema("bnpk::rows_kmer_table_insert", ""))
    for name in ("keys", "counts", "n_used"):
        assert re.search(rf"Tensor\([a-z]!\) {name}", schema), schema


def test_table_kernels_are_sm90a_code_without_stack():
    """Every build of the table mode of the row kernel, and the rehash kernel, is sm_90a SASS without local memory."""
    from bionumpy_b200 import _native
    tool = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(tool):
        pytest.skip("cuobjdump not available")
    out = subprocess.run([tool, "-res-usage", _native.LIB_PATH], capture_output=True, text=True).stdout
    assert "sm_90a" in out
    blocks = out.split(" Function ")
    names = ["_ZN4bnpk11rows_kernelILi5ELi%dELb0ELb0EEEvNS_7RowArgsE" % enc for enc in range(4)]
    names.append("_ZN4bnpk19table_rehash_kernelEPKlS1_mNS_9KmerTableEPl")
    for name in names:
        blk = next((b for b in blocks if b.startswith(name)), None)
        assert blk is not None, name
        m = re.search(r"REG:(\d+) STACK:(\d+)", blk)
        assert m and int(m.group(2)) == 0, (name, m and m.group(0))


# ---------------------------------------------------------------------------------------------------------------
# GPU: results against the oracle
# ---------------------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("k", [1, 5, 16, 21, 31])
@pytest.mark.parametrize("alphabet", ["ACGT", "ACTG"])
@pytest.mark.parametrize("canonical", [False, True])
def test_random_ragged_rows(bnp, k, alphabet, canonical):
    rng = np.random.default_rng(k * 7 + len(alphabet) + canonical)
    strings = random_rows(rng, 300, 120)
    enc = bnp.DNAEncoding if alphabet == "ACGT" else bnp.ACTGEncoding
    seqs = bnp.as_encoded_array(strings, enc)
    got = bnp.count_kmers_exact(seqs, k, canonical=canonical)
    assert_table(got, oracle_table(strings, k, canonical, alphabet))
    if alphabet == "ACGT":
        # BaseEncoding text is read as DNAEncoding, like get_kmers
        assert_table(bnp.count_kmers_exact(bnp.as_encoded_array(strings), k, canonical=canonical),
                     oracle_table(strings, k, canonical, alphabet))


@gpu
def test_batches_split_by_rows_when_the_table_is_small(bnp, monkeypatch):
    """A small minimum batch makes every add run as several row batches and several rehashes."""
    from bionumpy_b200.sequence import exact_counts as ec
    monkeypatch.setattr(ec, "MIN_BATCH", 500)
    rng = np.random.default_rng(5)
    strings = random_rows(rng, 400, 150)
    counter = bnp.KmerCounter(11, capacity=4)
    counter.add(bnp.as_encoded_array(strings))
    assert counter.n_grows >= 3
    assert_table(counter.result(), oracle_table(strings, 11))


@gpu
def test_fastq_stream_and_counter_equal_the_whole_file(bnp, tmp_path):
    rng = np.random.default_rng(3)
    text = make_fastq(rng, 700, min_len=0, max_len=180, lower_frac=0.1)
    path = tmp_path / "reads.fq"
    path.write_bytes(text.tobytes())
    size, starts, lens = oracle.fastq_split(text)
    seq_rows = [text[s:s + L].tobytes().decode() for s, L in zip(starts[:, 1], lens[:, 1])]
    for k, canonical in ((21, False), (31, True), (4, False)):
        want = oracle_table(seq_rows, k, canonical)
        got = bnp.count_kmers_exact(bnp.open(str(path)).read_chunks(min_chunk_size=5000), k, canonical=canonical)
        assert_table(got, want)
        counter = bnp.KmerCounter(k, canonical=canonical, capacity=100)
        n_chunks = 0
        for chunk in bnp.open(str(path)).read_chunks(min_chunk_size=3000):
            counter.add(chunk.sequence)
            n_chunks += 1
        assert n_chunks > 10
        assert_table(counter.result(), want)
        # the table stays usable: adding the file again doubles every count
        for chunk in bnp.open(str(path)).read_chunks(min_chunk_size=20000):
            counter.add(chunk)
        again = counter.result()
        assert np.array_equal(again.kmers.cpu().numpy(), want[0]) and np.array_equal(again.counts.cpu().numpy(), 2 * want[1])


@gpu
def test_saccer3_whole_genome_k21(bnp, tmp_path):
    """The reference's own sacCer3.fa: 17 chromosome-length rows (cut into warp-sized pieces), k = 21."""
    raw = gzip.open(os.path.join(ROOT, "tests", "golden", "sacCer3.fa.gz")).read()
    path = tmp_path / "sacCer3.fa"
    path.write_bytes(raw)
    whole = np.frombuffer((raw if raw.endswith(b"\n") else raw + b"\n") + b">", dtype=np.uint8)
    size, hs, hl, flat, seq_lens = oracle.multiline_fasta_split(whole)
    codes = oracle.encode_flat(flat, oracle.alphabet_lut("ACGT"))
    want_h, _ = oracle.get_kmers(codes, seq_lens, 21)
    u_want, c_want = np.unique(want_h, return_counts=True)
    chunk = bnp.open(str(path)).read()
    got = bnp.count_kmers_exact(chunk.sequence, 21, capacity=12_000_000)
    assert np.array_equal(got.kmers.cpu().numpy(), u_want) and np.array_equal(got.counts.cpu().numpy(), c_want)
    streamed = bnp.count_kmers_exact(bnp.open(str(path)).read_chunks(min_chunk_size=3_000_000), 21)
    assert np.array_equal(streamed.kmers.cpu().numpy(), u_want) and np.array_equal(streamed.counts.cpu().numpy(), c_want)
    assert int(got.counts.sum()) == want_h.size


@gpu
def test_growth_from_a_tiny_table_equals_a_presized_one(bnp):
    rng = np.random.default_rng(9)
    chunks = [random_rows(rng, 60, 200) for _ in range(12)]
    small = bnp.KmerCounter(25, canonical=True, capacity=16)
    big = bnp.KmerCounter(25, canonical=True, capacity=100_000)
    assert small.capacity == 32
    caps = []
    for strings in chunks:
        seqs = bnp.as_encoded_array(strings)
        small.add(seqs)
        big.add(seqs)
        caps.append(small.capacity)
    assert small.n_grows >= 3 and big.n_grows == 0 and caps == sorted(caps)
    a, b = small.result(), big.result()
    assert torch.equal(a.kmers, b.kmers) and torch.equal(a.counts, b.counts)
    assert_table(a, oracle_table(sum(chunks, []), 25, canonical=True))
    assert small.n_distinct == len(a) <= small.capacity // 2


@gpu
@pytest.mark.parametrize("k", [1, 7, 31])
def test_one_key_under_heavy_contention(bnp, k):
    strings = ["A" * 5000] * 40 + ["ACG" * 2000] * 40 + ["AC" * 3000] * 40
    for canonical in (False, True):
        got = bnp.count_kmers_exact(bnp.as_encoded_array(strings), k, canonical=canonical)
        assert_table(got, oracle_table(strings, k, canonical))
        assert int(got.counts.sum()) == sum(max(len(s) - k + 1, 0) for s in strings)


@gpu
@pytest.mark.parametrize("k", [1, 3, 8])
def test_small_k_matches_the_exact_histogram(bnp, k):
    rng = np.random.default_rng(k)
    seqs = bnp.as_encoded_array(random_rows(rng, 200, 90), bnp.DNAEncoding)
    got = bnp.count_kmers_exact(seqs, k)
    dense = torch.zeros(4 ** k, dtype=torch.int64, device=got.kmers.device)
    dense[got.kmers] = got.counts
    assert torch.equal(dense, bnp.count_kmers(seqs, k, axis=None).counts)


@gpu
def test_bad_base_raises_like_get_kmers_and_the_counter_refuses(bnp):
    strings = ["ACGTACGTAC", "ACGTT", "AC" * 9000 + "N" + "ACGT" * 10, "ACGNT"]
    seqs = bnp.as_encoded_array(strings)
    with pytest.raises(bnp.EncodingError) as want:
        bnp.get_kmers(seqs, 5).raw()
    with pytest.raises(bnp.EncodingError) as got:
        bnp.count_kmers_exact(seqs, 5)
    assert got.value.offset == want.value.offset == 15 + 18000
    counter = bnp.KmerCounter(5)
    counter.add(bnp.as_encoded_array(strings[:2]))
    with pytest.raises(bnp.EncodingError) as got:
        counter.add(seqs)
    assert got.value.offset == want.value.offset
    with pytest.raises(RuntimeError, match="failed earlier"):
        counter.add(bnp.as_encoded_array(strings[:2]))
    with pytest.raises(RuntimeError, match="failed earlier"):
        counter.result()
    with pytest.raises(NotImplementedError):
        bnp.count_kmers_exact(bnp.as_encoded_array(["MKV"], bnp.AminoAcidEncoding), 2)


@gpu
def test_lookups_most_common_and_spectrum(bnp):
    strings = ["ACGTACGTAA", "ACGTT", "TTTTTTT", "CC", ""]
    got = bnp.count_kmers_exact(bnp.as_encoded_array(strings), 3)
    u, c = oracle_table(strings, 3)
    assert_table(got, (u, c))
    assert got["ACG"] == 3 and got["TTT"] == 5 and got["GGG"] == 0 and got["acg"] == 3
    labels = [oracle.kmer_to_string(int(h), 3) for h in u]
    assert got.get_counts(labels + ["CCC"]).cpu().tolist() == c.tolist() + [0]
    assert got.get_counts(torch.tensor(u)).cpu().tolist() == c.tolist()
    kmers, counts = got.most_common()
    order = np.lexsort((u, -c))                                 # count descending, then k-mer ascending
    assert kmers.cpu().tolist() == u[order].tolist() and counts.cpu().tolist() == c[order].tolist()
    k2, c2 = got.most_common(2)
    assert k2.cpu().tolist() == u[order][:2].tolist()
    for max_count in (1, 2, 3, 10):
        want = np.bincount(np.minimum(c, max_count), minlength=max_count + 1)
        assert got.spectrum(max_count).cpu().tolist() == want.tolist()
    canon = bnp.count_kmers_exact(bnp.as_encoded_array(strings), 3, canonical=True)
    assert canon["ACG"] == canon["CGT"] == 6 and canon["AAA"] == canon["TTT"] == 5
    empty = bnp.KmerCounter(9).result()
    assert len(empty) == 0 and empty["ACGTACGTA"] == 0


@gpu
def test_dispatcher_op_matches_the_ctypes_path(bnp):
    from bionumpy_b200 import _native as nv, ops, torch_ops
    tops = torch_ops.load()
    rng = np.random.default_rng(4)
    strings = random_rows(rng, 150, 100)
    src = bnp.sequence.kmers._source_of(bnp.as_encoded_array(strings))
    base, starts, lens = src.base, src.starts, src.lens
    for cx in (0, 3):
        tables = []
        for via_torch in (False, True):
            keys = torch.full((1 << 15,), -1, dtype=torch.int64, device="cuda")
            counts = torch.zeros_like(keys)
            n_used = torch.zeros(1, dtype=torch.int64, device="cuda")
            if via_torch:
                status = tops.rows_kmer_table_insert(base, starts, lens, nv.ENC_ASCII_ACGT, None, 13, cx, keys, counts, n_used)
            else:
                status = ops.rows_kmer_table_insert(base, starts, lens, nv.ENC_ASCII_ACGT, 13, keys, counts, n_used, cx)
            assert ops.read_status(status).bad_base() is None
            tables.append((keys.cpu(), counts.cpu(), int(n_used.item())))
        (k0, c0, n0), (k1, c1, n1) = tables
        assert torch.equal(k0 >= 0, k1 >= 0) and n0 == n1 == int((k0 >= 0).sum())
        u, c = oracle_table(strings, 13, canonical=bool(cx))
        for keys, counts in ((k0, c0), (k1, c1)):
            keep = keys >= 0
            order = torch.argsort(keys[keep])
            assert np.array_equal(keys[keep][order].numpy(), u) and np.array_equal(counts[keep][order].numpy(), c)
            assert int(counts[~keep].abs().sum()) == 0
