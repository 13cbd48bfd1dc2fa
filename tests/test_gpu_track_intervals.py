"""Tracks back into intervals on the GPU (bnpk_runs_to_intervals): GenomicIntervals.from_track, GenomicArray.get_data
and GenomicRunLengthArray.to_bedgraph, each against tests/delimited_write_oracle.py, which sees only dense arrays."""
import gzip
import os
import warnings

import numpy as np
import pytest
import torch

import bionumpy_b200 as bnp
from bionumpy_b200 import _native as nv
from bionumpy_b200 import ops, torch_ops
from bionumpy_b200.arithmetics import GenomicRunLengthArray
from bionumpy_b200.genomic_data import keep_all

import delimited_write_oracle as wo
import pileup_oracle as po

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
TILE = 2048
DTYPES = [np.bool_, np.int8, np.uint8, np.int32, np.int64]


def _genome_track(sizes, dense, filter_function=keep_all, dtype=None):
    """A GenomicArray whose global dense values are ``dense`` (the kept contigs end to end), and the dense array of
    every kept contig."""
    genome = bnp.Genome.from_dict(sizes, filter_function=filter_function)
    dense = np.asarray(dense)
    assert dense.size == genome.size
    s, e, v = po.runs_of(dense)
    events = torch.from_numpy(np.concatenate([s, [dense.size]]).astype(np.int64)).cuda()
    values = torch.from_numpy(np.asarray(v, dtype=dtype or dense.dtype)).cuda()
    per_contig, off = {}, 0
    for name, size in genome.chrom_sizes.items():
        per_contig[name] = dense[off:off + size]
        off += size
    return bnp.GenomicArray(events, values, genome), per_contig


def _rows(record):
    return record.chromosome.tolist(), record.start.cpu().numpy(), record.stop.cpu().numpy()


def _check_intervals(iv, per_contig):
    names, starts, stops = wo.nonzero_intervals(per_contig)
    got = _rows(iv.get_data())
    assert got[0] == names
    assert got[1].tolist() == starts.tolist() and got[2].tolist() == stops.tolist()
    offsets = np.cumsum([0] + [len(d) for d in per_contig.values()])[:-1]
    off = dict(zip(per_contig, offsets.tolist()))
    glob = np.array([off[n] for n in names], dtype=np.int64)
    assert iv._g_start.cpu().tolist() == (starts + glob).tolist()
    assert iv._g_stop.cpu().tolist() == (stops + glob).tolist()
    assert [iv._genome._name_table()[0][i] for i in iv._ids.cpu().tolist()] == names


def _check_bedgraph(bg, per_contig, dtype):
    names, starts, stops, values = wo.bedgraph_rows(per_contig)
    got = _rows(bg)
    assert got[0] == names and got[1].tolist() == starts.tolist() and got[2].tolist() == stops.tolist()
    assert bg.value.dtype == torch.from_numpy(np.zeros(0, dtype)).dtype
    assert bg.value.cpu().numpy().astype(np.int64).tolist() == values.tolist()


def _random_dense(rng, n, dtype, max_run=6, p_zero=0.4):
    lens = rng.integers(1, max_run + 1, n)
    if dtype == np.bool_:
        vals = rng.random(lens.size) > p_zero
    else:
        info = np.iinfo(dtype)
        vals = rng.integers(max(info.min, -100), min(info.max, 100), lens.size, endpoint=True).astype(dtype)
        vals[rng.random(lens.size) < p_zero] = 0
    return np.repeat(vals, lens)[:n]


# --------------------------------------------------------------------------------------------------------------------
# every value type, runs on and across contig borders
# --------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", DTYPES)
def test_from_track_and_get_data_every_dtype(dtype):
    rng = np.random.default_rng(DTYPES.index(dtype))
    sizes = {"chr1": 5000, "s1": 1, "s2": 3, "empty": 0, "chr2": 7000, "s3": 2, "chr3": 333}
    dense = _random_dense(rng, sum(sizes.values()), dtype)
    track, per_contig = _genome_track(sizes, dense)
    _check_intervals(bnp.GenomicIntervals.from_track(track), per_contig)
    data = track.get_data()
    if dtype == np.bool_:
        assert isinstance(data, bnp.Interval)
        names, starts, stops = wo.nonzero_intervals(per_contig)
        assert _rows(data)[0] == names and _rows(data)[1].tolist() == starts.tolist()
    else:
        assert isinstance(data, bnp.BedGraph)
        _check_bedgraph(data, per_contig, dtype)


@pytest.mark.parametrize("where", ["start", "end", "span", "many"])
def test_runs_on_contig_borders(where):
    sizes = {f"c{i}": s for i, s in enumerate([10, 1, 1, 5, 0, 2, 1, 20])}
    n = sum(sizes.values())
    dense = np.zeros(n, dtype=np.int64)
    if where == "start":          # runs that begin exactly at contig starts
        dense[10:12] = 3
        dense[17:19] = 4
    elif where == "end":          # runs that end exactly at contig ends
        dense[5:10] = 2
        dense[12:17] = 5
    elif where == "span":         # one run from inside c0 to inside c7
        dense[4:30] = 7
    else:                         # a value change at every position
        dense[:] = np.arange(n) % 3
    track, per_contig = _genome_track(sizes, dense)
    _check_intervals(bnp.GenomicIntervals.from_track(track), per_contig)
    _check_bedgraph(track.get_data(), per_contig, np.int64)
    mask, pc = _genome_track(sizes, dense != 0)
    _check_intervals(bnp.GenomicIntervals.from_track(mask), pc)


def test_all_zero_run_over_hundreds_of_scaffolds():
    sizes = {"chr1": 100, **{f"scaffold_{i}": 1 + i % 7 for i in range(300)}, "chr2": 50}
    dense = np.zeros(sum(sizes.values()), dtype=np.int32)
    dense[:60] = 1
    dense[-10:] = 2
    track, per_contig = _genome_track(sizes, dense)
    bg = track.get_data()
    assert len(bg) == 2 + 300 + 2
    _check_bedgraph(bg, per_contig, np.int32)
    _check_intervals(bnp.GenomicIntervals.from_track(track), per_contig)


def test_left_out_contigs_on_hg38_names():
    """hg38's contigs in file order, a ten-thousandth of their sizes: the contigs with '_' (ignore_underscores) are
    left out of the layout, and so are the rows on them."""
    sizes = po.read_sizes(open(os.path.join(GOLDEN, "hg38.chrom.sizes")).read())
    sizes = {n: s // 10000 for n, s in sizes.items()}
    keep = {n: s for n, s in sizes.items() if "_" not in n}
    assert 0 in sizes.values() and len(keep) < len(sizes)
    rng = np.random.default_rng(3)
    track, per_contig = _genome_track(sizes, _random_dense(rng, sum(keep.values()), np.int64, max_run=40),
                                      filter_function=lambda n: "_" not in n)
    assert list(per_contig) == list(keep)
    iv = bnp.GenomicIntervals.from_track(track)
    assert not any("_" in n for n in iv.get_data().chromosome.tolist())
    _check_intervals(iv, per_contig)
    _check_bedgraph(track.get_data(), per_contig, np.int64)


# --------------------------------------------------------------------------------------------------------------------
# non-canonical and degenerate tracks, tile borders
# --------------------------------------------------------------------------------------------------------------------
def test_non_canonical_tracks_from_astype():
    sizes = {"a": 40, "b": 30}
    dense = np.repeat(np.array([0, 256, 512, 1, 257, 0, 3, 259, 0], dtype=np.int64), [5, 5, 5, 5, 10, 5, 15, 15, 5])
    track, _ = _genome_track(sizes, dense)
    narrow = bnp.GenomicArray._of(track._global.astype(torch.int8), track._genome)      # 0, 0, 0, 1, 1, 0, 3, 3, 0
    per_contig = {"a": dense[:40].astype(np.int8), "b": dense[40:].astype(np.int8)}
    assert narrow._global.values.numel() == 9                                          # equal neighbours kept
    _check_intervals(bnp.GenomicIntervals.from_track(narrow), per_contig)
    bg = narrow.get_data()                                                               # every stored run
    assert bg.value.dtype == torch.int8
    got = wo.dense_of_rows(*_rows(bg), bg.value.cpu().numpy(), sizes, np.int8)
    for name in sizes:
        assert np.array_equal(got[name], per_contig[name])
    assert _rows(bg)[1].tolist() == [0, 5, 10, 15, 20, 30, 35, 0, 10, 25]


def test_all_zero_and_one_run_tracks():
    sizes = {"a": 1000, "b": 1, "c": 77}
    n = sum(sizes.values())
    zero, _ = _genome_track(sizes, np.zeros(n, np.int64))
    assert len(bnp.GenomicIntervals.from_track(zero)) == 0
    assert _rows(zero.get_data())[1].tolist() == [0, 0, 0]
    ones, pc = _genome_track(sizes, np.ones(n, np.bool_))
    iv = bnp.GenomicIntervals.from_track(ones)
    assert _rows(iv.get_data())[0] == ["a", "b", "c"]
    _check_intervals(iv, pc)
    empty = bnp.Genome.from_dict({"x": 0})
    none = bnp.GenomicArray(torch.zeros(2, dtype=torch.int64, device="cuda"),
                            torch.zeros(1, dtype=torch.int64, device="cuda"), empty)
    assert len(bnp.GenomicIntervals.from_track(none)) == 0 and len(none.get_data()) == 0


@pytest.mark.parametrize("n_runs", [TILE - 1, TILE, TILE + 1, 2 * TILE - 8, 2 * TILE + 7, 300 * TILE + 5])
def test_row_counts_around_tile_borders(n_runs):
    rng = np.random.default_rng(n_runs)
    lens = rng.integers(1, 5, n_runs)
    values = rng.integers(0, 3, n_runs)
    values[1:][values[1:] == values[:-1]] += 3                      # canonical runs
    dense = np.repeat(values, lens).astype(np.int64)
    cut = np.sort(rng.choice(np.arange(1, dense.size), 40, replace=False))
    sizes = {f"c{i}": int(b - a) for i, (a, b) in enumerate(zip(np.concatenate([[0], cut]),
                                                                 np.concatenate([cut, [dense.size]])))}
    track, per_contig = _genome_track(sizes, dense)
    _check_intervals(bnp.GenomicIntervals.from_track(track), per_contig)
    _check_bedgraph(track.get_data(), per_contig, np.int64)


def test_kernel_directly_with_ends_beyond_shared_memory():
    """More than 2047 contigs: the ends are searched in global memory."""
    rng = np.random.default_rng(9)
    ends = np.concatenate([[0], np.cumsum(rng.integers(1, 4, 3000))]).astype(np.int64)
    size = int(ends[-1])
    dense = (rng.random(size) < 0.5).astype(np.int64) * rng.integers(1, 3, size)
    s, e, v = po.runs_of(dense)
    ev = torch.from_numpy(np.concatenate([s, [size]])).cuda()
    vals = torch.from_numpy(v.astype(np.int64)).cuda()
    for mode in (nv.RUNS_TO_NONZERO, nv.RUNS_TO_ALL):
        contig, start, stop, value, n_out = ops.runs_to_intervals(ev, vals, torch.from_numpy(ends).cuda(), mode)
        k = int(n_out.item())
        per_contig = {i: dense[ends[i]:ends[i + 1]] for i in range(len(ends) - 1)}
        if mode == nv.RUNS_TO_NONZERO:
            names, ws, we = wo.nonzero_intervals(per_contig)
        else:
            names, ws, we, wv = wo.bedgraph_rows(per_contig)
            assert value[:k].cpu().tolist() == wv.tolist()
        glob = ends[np.array(names, dtype=np.int64)] if names else np.zeros(0, np.int64)
        assert contig[:k].cpu().tolist() == names
        assert start[:k].cpu().tolist() == (ws + glob).tolist() and stop[:k].cpu().tolist() == (we + glob).tolist()
    # the dispatcher op gives the same rows
    c2, s2, e2, v2, n2 = torch_ops.load().runs_to_intervals(ev, vals, torch.from_numpy(ends).cuda(), nv.RUNS_TO_ALL)
    assert int(n2.item()) == k and torch.equal(s2[:k], start[:k]) and torch.equal(v2[:k], value[:k])


def test_to_bedgraph():
    dense = np.array([0, 0, 3, 3, 1, 0, 0, 0, 2], dtype=np.int32)
    s, e, v = po.runs_of(dense)
    track = GenomicRunLengthArray.from_runs(s, e, torch.from_numpy(v))
    bg = track.to_bedgraph("chr10")
    assert bg.chromosome.tolist() == ["chr10"] * 5
    assert _rows(bg)[1].tolist() == s.tolist() and _rows(bg)[2].tolist() == e.tolist()
    assert bg.value.dtype == torch.int32 and bg.value.cpu().tolist() == v.tolist()
    mask = GenomicRunLengthArray.from_runs([0, 4], [4, 9], torch.tensor([False, True]))
    out = bnp.io.BdgBuffer.from_data(mask.to_bedgraph("m")).raw().cpu().numpy().tobytes()
    assert out == b"m\t0\t4\t0\nm\t4\t9\t1\n"                       # bool values as 0 / 1


# --------------------------------------------------------------------------------------------------------------------
# hg38 peaks, round trip through a BED file
# --------------------------------------------------------------------------------------------------------------------
def test_znf263_mask_round_trip_on_hg38(tmp_path):
    """from_track of the peaks' mask is the peaks merged on every contig (touching peaks merge, as in the mask), in
    genome order; written as BED and read back it gives the same mask."""
    hg38 = bnp.Genome.from_file(os.path.join(GOLDEN, "hg38.chrom.sizes"))
    mask = hg38.read_intervals(os.path.join(GOLDEN, "znf263.bed.gz")).get_mask()
    iv = bnp.GenomicIntervals.from_track(mask)
    chroms, starts, stops = po.parse_bed(gzip.open(os.path.join(GOLDEN, "znf263.bed.gz")).read())
    order = {n: i for i, n in enumerate(hg38.chrom_sizes)}
    rows = sorted((order[c], a, b, c) for c, a, b in zip(chroms, starts, stops) if c in order and b > a)
    names = [r[3] for r in rows]
    s = np.array([r[1] for r in rows], dtype=np.int64)
    first, merged_stops = po.merge_by_chromosome(names, s, np.array([r[2] for r in rows], dtype=np.int64))
    want_names, want_starts = [names[i] for i in first], s[first]
    got = _rows(iv.get_data())
    assert got[0] == want_names and got[1].tolist() == want_starts.tolist() and got[2].tolist() == merged_stops.tolist()
    # a small contig against its dense mask
    d = po.dense_mask(s[np.array(names) == "chr21"], np.array([r[2] for r in rows])[np.array(names) == "chr21"],
                      hg38.chrom_sizes["chr21"])
    w = wo.nonzero_intervals({"chr21": d})
    sel = np.array(got[0]) == "chr21"
    assert got[1][sel].tolist() == w[1].tolist() and got[2][sel].tolist() == w[2].tolist()
    path = str(tmp_path / "peaks.bed")
    with bnp.open(path, "w", buffer_type=bnp.io.BedBuffer) as f:
        f.write(iv.get_data())
    assert open(path, "rb").read() == wo.dump_lines(wo.bed_columns(want_names, want_starts, merged_stops))
    back = hg38.read_intervals(path).get_mask()
    assert int((mask ^ back).sum()) == 0
    assert int((iv.merged().get_mask() ^ mask).sum()) == 0 and len(iv.sorted()) == len(iv)
    assert bool(mask[iv].min().all())


# --------------------------------------------------------------------------------------------------------------------
# synchronisations and launches
# --------------------------------------------------------------------------------------------------------------------
def _count_syncs(fn):
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("warn")
    try:
        with warnings.catch_warnings(record=True) as caught:
            warnings.simplefilter("always")
            out = fn()
    finally:
        torch.cuda.set_sync_debug_mode(0)
    return out, len([w for w in caught if "synchroniz" in str(w.message)])


def test_one_synchronisation_and_fixed_launches():
    lib = nv.load_library()
    sizes = {"chr1": 3_000_000, "chr2": 1000, "chrX": 500}
    seen = {}
    for n in (10, 200_000):
        rng = np.random.default_rng(n)
        dense = np.zeros(sum(sizes.values()), dtype=np.int64)
        idx = rng.integers(0, dense.size, n)
        dense[idx] = rng.integers(1, 5, n)
        track, _ = _genome_track(sizes, dense)
        mask = track > 0
        bnp.GenomicIntervals.from_track(mask)                                  # the genome's tables are built once
        for name, fn in (("from_track", lambda: bnp.GenomicIntervals.from_track(mask)),
                         ("get_data", lambda: track.get_data()), ("mask_data", lambda: mask.get_data())):
            before = lib.bnpk_launch_count()
            _, syncs = _count_syncs(fn)
            seen.setdefault(name, set()).add(lib.bnpk_launch_count() - before)
            assert syncs == 1, (name, syncs)
    assert all(len(v) == 1 for v in seen.values()), seen
