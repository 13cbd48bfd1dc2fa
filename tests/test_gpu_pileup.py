"""Pileups, masks, merges and run-length tracks on the GPU against the NumPy oracle (tests/pileup_oracle.py): every run,
value, row and byte must equal the oracle's."""
import gzip
import os
import warnings

import numpy as np
import pytest
import torch

import bionumpy_b200 as bnp
from bionumpy_b200 import _native as nv
from bionumpy_b200 import ops
from bionumpy_b200.arithmetics import get_pileup, get_boolean_mask, merge_intervals
from bionumpy_b200.ragged import RaggedArray

import pileup_oracle as po

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
TILE = 2048                      # event keys per tile of pileup_runs_kernel / rows per tile of the merge


def _iv(starts, stops, chrom="chr1"):
    starts, stops = np.asarray(starts, dtype=np.int64), np.asarray(stops, dtype=np.int64)
    names = chrom if isinstance(chrom, list) else [chrom] * len(starts)
    return bnp.Interval(names, starts, stops)


def _check_runs(arr, starts, stops, size, any_mode=False):
    s, e, v = po.event_runs(starts, stops, size, any_mode)
    assert len(arr) == size
    assert arr.starts.cpu().numpy().tolist() == s.tolist()
    assert arr.ends.cpu().numpy().tolist() == e.tolist()
    assert arr.values.cpu().numpy().tolist() == v.tolist()
    assert arr.values.dtype == (torch.bool if any_mode else torch.int64)


def _both(starts, stops, size):
    _check_runs(get_pileup(_iv(starts, stops), size), starts, stops, size)
    _check_runs(get_boolean_mask(_iv(starts, stops), size), starts, stops, size, True)


def test_docstrings():
    iv = _iv([3, 5, 10], [8, 7, 12])
    assert str(get_pileup(iv, 20)) == "[0 0 0 1 1 2 2 1 0 0 1 1 0 0 0 0 0 0 0 0]"
    mask = get_boolean_mask(iv, 20)
    assert str(mask.astype(int)) == "[0 0 0 1 1 1 1 1 0 0 1 1 0 0 0 0 0 0 0 0]"
    other = get_boolean_mask(_iv([9], [15]), 20)
    assert other[iv.start].cpu().tolist() == [False, False, True]


@pytest.mark.parametrize("n", [0, 1, 2])
def test_few_intervals(n):
    starts, stops = np.array([4, 2][:n]), np.array([9, 6][:n])
    _both(starts, stops, 20)


@pytest.mark.parametrize("tiles", [1, 2, 3])
@pytest.mark.parametrize("delta", [-1, 0, 1])
def test_tile_borders(tiles, delta):
    """2n event keys one tile -1 / 0 / +1 around the first tile borders, on few positions, so groups of equal
    positions straddle the borders."""
    rng = np.random.default_rng(tiles * 3 + delta)
    n = (tiles * TILE + 2 * delta) // 2
    a = rng.integers(0, 40, n)
    b = a + rng.integers(0, 5, n)
    _both(a, b, 50)


def test_one_million_random_intervals():
    rng = np.random.default_rng(1)
    n, size = 1_000_000, 10_000_000
    a = rng.integers(0, size, n)
    b = np.minimum(a + rng.integers(0, 2000, n), size)
    a[:1000], b[:1000] = a[1000:2000], b[1000:2000]                       # duplicates
    a[2000:3000], b[2000:3000] = a[1000:2000] + 1, np.maximum(b[1000:2000] - 1, a[1000:2000] + 1)   # nested
    _both(a, b, size)


def test_abutting_and_zero_length():
    arr = get_pileup(_iv([0, 5, 12], [5, 10, 12]), 20)
    assert arr.starts.cpu().tolist() == [0, 10] and arr.values.cpu().tolist() == [1, 0]
    _both([3, 3, 7], [3, 3, 7], 10)
    _both([0, 5, 5], [5, 5, 9], 9)


def test_same_start_and_same_stop_across_tiles():
    rng = np.random.default_rng(7)
    n = 10_000
    stops = 100 + rng.integers(0, 1000, n)
    _both(np.full(n, 100), stops, 2000)
    starts = rng.integers(0, 500, n)
    _both(starts, np.full(n, 500), 2000)
    _both(np.full(n, 0), np.full(n, 2000), 2000)


def test_contig_ends_and_size_one():
    _both([0], [1], 1)
    _both([], [], 1)
    _both([0, 5], [3, 10], 10)
    _both([9], [10], 10)


def test_to_array_and_indexing():
    rng = np.random.default_rng(2)
    a = rng.integers(0, 5000, 3000)
    b = np.minimum(a + rng.integers(0, 300, 3000), 5000)
    arr = get_pileup(_iv(a, b), 5000)
    dense = po.dense_pileup(a, b, 5000)
    assert arr.to_array().cpu().numpy().tolist() == dense.tolist()
    assert arr[17] == dense[17] and arr[-1] == dense[-1]
    sub = arr[1000:3000]
    assert sub.to_array().cpu().numpy().tolist() == dense[1000:3000].tolist() and len(sub) == 2000
    s, e, v = po.runs_of(dense[1000:3000])
    assert sub.starts.cpu().tolist() == s.tolist() and sub.values.cpu().tolist() == v.tolist()
    pos = rng.integers(0, 5000, 100)
    assert arr[torch.as_tensor(pos)].cpu().numpy().tolist() == dense[pos].tolist()
    assert int(arr.max()) == dense.max() and int(arr.sum()) == dense.sum()
    assert float(arr.mean()) == pytest.approx(dense.mean())


def _queries(rng, n, size, length=100):
    a = rng.integers(0, size - length, n)
    return a, a + length


def test_million_queries_fused_against_oracle():
    rng = np.random.default_rng(4)
    size = 10_000_000
    a = rng.integers(0, size, 1_000_000)
    b = np.minimum(a + 150, size)
    arr = get_pileup(_iv(a, b), size)
    dense = torch.as_tensor(po.dense_pileup(a, b, size))
    qa, qb = _queries(rng, 1_000_000, size)
    peaks = _iv(qa, qb)
    lazy = arr[peaks]
    got = {how: getattr(lazy, how)(axis=-1).cpu() for how in ("max", "min", "sum", "mean", "any")}
    assert not lazy.is_materialised()
    for lo in range(0, qa.size, 100_000):
        idx = torch.as_tensor(qa[lo:lo + 100_000])[:, None] + torch.arange(100)
        rows = dense[idx]
        assert torch.equal(got["max"][lo:lo + 100_000], rows.max(1).values)
        assert torch.equal(got["min"][lo:lo + 100_000], rows.min(1).values)
        assert torch.equal(got["sum"][lo:lo + 100_000], rows.sum(1))
        assert torch.allclose(got["mean"][lo:lo + 100_000], rows.double().mean(1))
        assert torch.equal(got["any"][lo:lo + 100_000], (rows != 0).any(1))
    # the fused and the materialised paths agree
    for how in ("max", "min", "sum", "any"):
        assert torch.equal(getattr(RaggedArray, how)(lazy, axis=-1).cpu().to(got[how].dtype), got[how]), how
    assert lazy.is_materialised()
    assert torch.equal(lazy.ravel().cpu(), dense[torch.as_tensor(qa)[:, None] + torch.arange(100)].reshape(-1))


def test_empty_queries_and_long_queries():
    """Empty rows follow RaggedArray; queries over more runs than a warp, a block and one grid's threads."""
    size = 2_000_000
    a = np.arange(0, size, 2)                   # 2 M runs of length 1 with values 1, 0, 1, ...
    arr = get_pileup(_iv(a, a + 1), size)
    assert arr.values.numel() == size
    qa = np.array([5, 0, 10, 100, 0, 7])
    qb = np.array([5, 40, 10 + 600, 100 + 40_000, size, 7])   # 40, 600, 40 k and 2 M runs
    lazy = arr[_iv(qa, qb)]
    mx, mn, sm = lazy.max(axis=-1).cpu(), lazy.min(axis=-1).cpu(), lazy.sum(axis=-1).cpu()
    dense = np.zeros(size, np.int64)
    dense[a] = 1
    for i, (s, e) in enumerate(zip(qa, qb)):
        if s == e:
            assert mx[i] == np.iinfo(np.int64).min and mn[i] == np.iinfo(np.int64).max and sm[i] == 0
        else:
            assert mx[i] == dense[s:e].max() and mn[i] == dense[s:e].min() and sm[i] == dense[s:e].sum()
    assert torch.isnan(lazy.mean(axis=-1)[0]) and not bool(lazy.any(axis=-1)[0])
    assert lazy.lengths.cpu().tolist() == (qb - qa).tolist()


def test_bounds_errors():
    for starts, stops, bad in (([1, -1, 2], [2, 3, 4], 1), ([1, 5, 2], [2, 3, 1], 1), ([1, 2, 3], [2, 3, 11], 2)):
        with pytest.raises(ValueError, match=f"interval {bad} "):
            get_pileup(_iv(starts, stops), 10)
        with pytest.raises(ValueError, match=f"interval {bad} "):
            get_boolean_mask(_iv(starts, stops), 10)


def test_genome_errors_and_dropped_contigs():
    g = bnp.Genome.from_file(os.path.join(GOLDEN, "hg38.chrom.sizes"))
    with pytest.raises(KeyError):
        g.get_intervals(_iv([1, 2], [3, 4], ["chr1", "chrNope"]))
    with pytest.raises(ValueError, match="interval 1 "):
        g.get_intervals(_iv([1, 2], [3, 248956423], ["chr1", "chr1"]))
    chroms = ["chr1", "chr1_KI270706v1_random", "chr2", "chrUn_GL000195v1", "chr2"]
    gi = g.get_intervals(_iv([1, 2, 3, 4, 5], [10, 20, 30, 40, 50], chroms))
    assert len(gi) == 3
    assert gi.start.cpu().tolist() == [1, 3, 5]


def test_multi_contig_genome_pileup():
    sizes = {"a": 10, "b_x": 4, "b": 1, "c": 7, "d": 5}
    g = bnp.Genome.from_dict(sizes, filter_function=lambda n: "_" not in n)
    chroms = ["a", "a", "b", "c", "c", "b_x", "a"]
    starts = np.array([0, 6, 0, 0, 3, 0, 9])
    stops = np.array([3, 10, 1, 2, 7, 4, 10])
    gi = g.get_intervals(_iv(starts, stops, chroms))
    keep, gs, ge = po.genome_intervals(sizes, chroms, starts, stops)
    names, offsets, total = po.genome_layout(sizes)
    for mode, track in ((False, gi.get_pileup()), (True, gi.get_mask())):
        s, e, v = po.event_runs(gs, ge, total, mode)
        assert track._global.starts.cpu().tolist() == s.tolist() and track._global.values.cpu().tolist() == v.tolist()
        for name in names:
            cs, ce, cv = po.contig_runs(s, e, v, offsets[name], sizes[name])
            got = track[name]
            assert got.starts.cpu().tolist() == cs.tolist() and got.ends.cpu().tolist() == ce.tolist()
            assert got.values.cpu().tolist() == cv.tolist() and len(got) == sizes[name]
    assert int(gi.get_pileup().sum()) == int((ge - gs).sum())
    # "d" has no interval: one zero run that spans the border from "c"
    assert gi.get_pileup()["d"].values.cpu().tolist() == [0]


def test_merge_distances():
    rng = np.random.default_rng(9)
    a = np.sort(rng.integers(0, 100_000, 20_000))
    b = a + rng.integers(0, 30, a.size)
    a[5:10] = a[4]                  # equal starts, zero-length rows
    b[5:10] = a[4]
    for d in (0, 1, 10 ** 9):
        got = merge_intervals(_iv(a, b), d)
        rows, stops = po.merge_intervals(a, b, d)
        assert got.start.cpu().tolist() == a[rows].tolist() and got.stop.cpu().tolist() == stops.tolist()
        assert type(got) is bnp.Interval


def test_merge_chromosome_changes_and_unsorted():
    chroms = ["chr1"] * 3 + ["chr2"] * 3 + ["chr10"] * 2
    a = np.array([5, 6, 8, 0, 7, 7, 1, 2])          # start falls where the chromosome changes
    b = np.array([9, 7, 20, 9, 8, 9, 3, 5])
    got = merge_intervals(_iv(a, b, chroms))
    rows, stops = po.merge_by_chromosome(chroms, a, b)
    assert got.start.cpu().tolist() == a[rows].tolist() and got.stop.cpu().tolist() == stops.tolist()
    assert [c.to_string() for c in got.chromosome] == [chroms[r] for r in rows]
    with pytest.raises(AssertionError, match="sorted on start position"):
        merge_intervals(_iv([1, 5, 4], [2, 6, 7]))
    # the same rows across tile borders: every row of its own chromosome, then one chromosome
    n = 3 * TILE + 5
    a = np.arange(n) * 2
    names = ["c%d" % (i // 7) for i in range(n)]
    got = merge_intervals(_iv(a, a + 3, names))
    rows, stops = po.merge_by_chromosome(names, a, a + 3)
    assert got.start.cpu().tolist() == a[rows].tolist() and got.stop.cpu().tolist() == stops.tolist()


@pytest.mark.parametrize("offset", range(16))
def test_rows_equal_prev_prefix_names(offset):
    """Neighbouring names that are prefixes of each other or differ in length, at view offsets 0..15."""
    names = [b"chr1", b"chr1", b"chr10", b"chr1", b"chr", b"chr", b"", b"", b"chr2", b"chr21", b"chr21"]
    text = b"#" * offset + b"".join(names)
    base = torch.frombuffer(bytearray(text + b"\xff" * 16), dtype=torch.uint8).cuda()
    lens = np.array([len(n) for n in names])
    starts = offset + np.concatenate([[0], np.cumsum(lens)[:-1]])
    flag = ops.rows_equal_prev(base, torch.as_tensor(starts).cuda(), torch.as_tensor(lens, dtype=torch.int32).cuda())
    want = [0] + [int(names[i] == names[i - 1]) for i in range(1, len(names))]
    assert flag.cpu().tolist() == want


def test_ctcf_on_hg38():
    g = bnp.Genome.from_file(os.path.join(GOLDEN, "hg38.chrom.sizes"))
    gi = g.read_intervals(os.path.join(GOLDEN, "ctcf.bed.gz"))
    chroms, starts, stops = po.parse_bed(gzip.open(os.path.join(GOLDEN, "ctcf.bed.gz")).read())
    sizes = po.read_sizes(open(os.path.join(GOLDEN, "hg38.chrom.sizes")).read())
    keep, gs, ge = po.genome_intervals(sizes, chroms, starts, stops)
    assert 0 < len(gi) == keep.size < len(chroms)
    _, _, total = po.genome_layout(sizes)
    for mode, track in ((False, gi.get_pileup()), (True, gi.get_mask())):
        s, e, v = po.event_runs(gs, ge, total, mode)
        assert track._global.starts.cpu().tolist() == s.tolist() and track._global.values.cpu().tolist() == v.tolist()
    merged = gi.merged()
    order = np.argsort(gs, kind="stable")
    kc = [chroms[r] for r in keep[order]]
    rows, mstops = po.merge_by_chromosome(kc, gs[order], ge[order])
    assert merged._g_start.cpu().tolist() == gs[order][rows].tolist()
    assert merged._g_stop.cpu().tolist() == mstops.tolist()
    assert [c.to_string() for c in merged.chromosome] == [kc[r] for r in rows]


def test_peak_pileup_chain():
    """scripts/peak_pileup_example.py on ctcf_chr21-22.bed.gz with synthetic 150-bp reads as intervals."""
    g = bnp.Genome.from_file(os.path.join(GOLDEN, "chr21-22.chrom.sizes"))
    peaks = g.read_intervals(os.path.join(GOLDEN, "ctcf_chr21-22.bed.gz"))
    pchroms, pstarts, pstops = po.parse_bed(gzip.open(os.path.join(GOLDEN, "ctcf_chr21-22.bed.gz")).read())
    rng = np.random.default_rng(11)
    n = 200_000
    pick = rng.integers(0, len(pchroms), n)
    rs = np.maximum(pstarts[pick] + rng.integers(-200, 200, n), 0)
    rchroms = [pchroms[i] for i in pick]
    reads = g.get_intervals(_iv(rs, rs + 150, rchroms))
    pileup = reads.get_pileup()
    best = np.max(pileup[peaks], axis=-1)
    high = peaks[best > 4]
    sizes = po.read_sizes(open(os.path.join(GOLDEN, "chr21-22.chrom.sizes")).read())
    _, gs, ge = po.genome_intervals(sizes, rchroms, rs, rs + 150)
    _, ps, pe = po.genome_intervals(sizes, pchroms, pstarts, pstops)
    _, _, total = po.genome_layout(sizes)
    s, e, v = po.event_runs(gs, ge, total)
    want = po.reduce_runs(s, e, v, ps, pe, "max")
    assert best.cpu().numpy().tolist() == want.tolist()
    assert high.start.cpu().tolist() == pstarts[want > 4].tolist()


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


def test_synchronisations_and_launch_counts():
    g = bnp.Genome.from_dict({"chr1": 50_000_000, "chr2": 1000})
    lib = nv.load_library()
    launches = []
    for n in (10, 1_000_000):
        rng = np.random.default_rng(n)
        a = np.sort(rng.integers(0, 40_000_000, n))
        iv = _iv(a, a + 150)
        gi = g.get_intervals(iv)
        for fn in (lambda: get_pileup(iv, 50_000_000), lambda: get_boolean_mask(iv, 50_000_000), gi.get_pileup,
                   gi.get_mask, gi.merged, lambda: merge_intervals(iv)):
            before = lib.bnpk_launch_count()
            _, syncs = _count_syncs(fn)
            launches.append((n, lib.bnpk_launch_count() - before))
            assert syncs == 1, fn
        track = gi.get_pileup()
        lazy, syncs = _count_syncs(lambda: track[gi].max(axis=-1))
        assert syncs == 0
        arr = track["chr1"]
        _, syncs = _count_syncs(lambda: arr[iv].sum(axis=-1))
        assert syncs == 0
        _, syncs = _count_syncs(lambda: track[gi]._data)
        assert syncs == 1
    assert [c for n, c in launches if n == 10] == [c for n, c in launches if n == 1_000_000], launches


def test_two_streams():
    rng = np.random.default_rng(5)
    cases = []
    for _ in range(2):
        a = rng.integers(0, 1_000_000, 200_000)
        cases.append((a, a + rng.integers(0, 500, a.size)))
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    ivs = [_iv(a, b) for a, b in cases]
    torch.cuda.synchronize()
    with torch.cuda.stream(s1):
        r1 = get_pileup(ivs[0], 1_000_600)
    with torch.cuda.stream(s2):
        r2 = get_pileup(ivs[1], 1_000_600)
    torch.cuda.synchronize()
    for r, (a, b) in zip((r1, r2), cases):
        _check_runs(r, a, b, 1_000_600)


def test_dispatcher_ops():
    torch.ops.load_library(os.path.join(os.path.dirname(nv.LIB_PATH), "libbnpk_torch.so"))
    rng = np.random.default_rng(6)
    a = torch.as_tensor(rng.integers(0, 10_000, 5000)).cuda()
    b = a + torch.as_tensor(rng.integers(0, 100, 5000)).cuda()
    keys, status = torch.ops.bnpk.interval_events(a, b, None, None, None, 10_100)
    keys2, _, _, _ = ops.interval_events(a, b, size=10_100)
    assert torch.equal(keys, keys2) and int(status[nv.ST_BAD_BASE]) == nv.INT64_MAX
    sk = torch.sort(keys).values
    runs = torch.ops.bnpk.pileup_runs(sk, 10_100, nv.PILEUP_COUNT)
    runs2 = ops.pileup_runs(sk, 10_100, nv.PILEUP_COUNT)
    n = int(runs[2][0])
    assert n == int(runs2[2][0]) and torch.equal(runs[0][:n + 1], runs2[0][:n + 1])
    assert torch.equal(runs[1][:n], runs2[1][:n])
    ev, vals = runs[0][:n + 1].contiguous(), runs[1][:n].contiguous()
    qa, qb = a[:100].contiguous(), b[:100].contiguous()
    for mode in (nv.RUNS_MAX, nv.RUNS_MIN, nv.RUNS_SUM, nv.RUNS_ANY):
        assert torch.equal(torch.ops.bnpk.runs_reduce(ev, vals, qa, qb, mode), ops.runs_reduce(ev, vals, qa, qb, mode))
    offs = ops.row_offsets((qb - qa).to(torch.int32))
    total = int(offs[-1])
    assert torch.equal(torch.ops.bnpk.runs_extract(ev, vals, qa, offs, total), ops.runs_extract(ev, vals, qa, offs, total))
    sa = torch.sort(a).values
    m1 = torch.ops.bnpk.interval_merge(sa, sa + 5, None, 2)
    m2 = ops.interval_merge(sa, sa + 5, None, 2)
    k = int(m1[2][0])
    assert k == int(m2[2][0]) and torch.equal(m1[0][:k], m2[0][:k]) and torch.equal(m1[1][:k], m2[1][:k])
    base = torch.frombuffer(bytearray(b"chr1chr1chr2"), dtype=torch.uint8).cuda()
    st = torch.tensor([0, 4, 8], device="cuda")
    ln = torch.tensor([4, 4, 4], dtype=torch.int32, device="cuda")
    assert torch.ops.bnpk.rows_equal_prev(base, st, ln).cpu().tolist() == [0, 1, 0]


@pytest.mark.parametrize("distance", [0, 1])
def test_merge_without_chromosome_flags(distance):
    """same_prev = None is one segment: the merge equals the oracle's across tile borders, and a start that decreases
    anywhere is reported."""
    torch.ops.load_library(os.path.join(os.path.dirname(nv.LIB_PATH), "libbnpk_torch.so"))
    rng = np.random.default_rng(20 + distance)
    n = 3 * TILE + 5
    a = np.sort(rng.integers(0, 4 * n, n))
    b = a + rng.integers(0, 6, n)
    ta, tb = torch.as_tensor(a).cuda(), torch.as_tensor(b).cuda()
    for first, stops, n_out, status in (ops.interval_merge(ta, tb, None, distance),
                                        torch.ops.bnpk.interval_merge(ta, tb, None, distance)):
        k = int(n_out[0])
        rows, want = po.merge_intervals(a, b, distance)
        assert k == rows.size < n
        assert first[:k].cpu().tolist() == rows.tolist() and stops[:k].cpu().tolist() == want.tolist()
        assert int(status[nv.ST_BAD_BASE]) == nv.INT64_MAX
    a2 = a.copy()
    a2[TILE + 3] = a2[TILE + 2] - 1                 # one row out of order, just past the first tile border
    a2[2 * TILE + 9] = -1
    _, _, _, status = ops.interval_merge(torch.as_tensor(a2).cuda(), tb, None, distance)
    assert int(status[nv.ST_BAD_BASE]) == TILE + 3


def test_merge_numpy_chromosome_names():
    """Chromosome names that are not device text (a NumPy array of str) are moved to the device first."""
    chroms = np.array(["chr1", "chr1", "chr1", "chr2", "chr2"])
    a, b = np.array([1, 3, 10, 0, 2]), np.array([5, 4, 12, 3, 4])
    got = merge_intervals(bnp.Interval(chroms, a, b))
    rows, stops = po.merge_by_chromosome(list(chroms), a, b)
    assert got.start.cpu().tolist() == a[rows].tolist() and got.stop.cpu().tolist() == stops.tolist()
    assert [c.to_string() for c in got.chromosome] == [chroms[r] for r in rows]
    with pytest.raises(AssertionError, match="sorted on start position"):
        merge_intervals(bnp.Interval(np.array(["chr1", "chr1"]), np.array([5, 1]), np.array([6, 2])))


def test_intervals_outside_the_track_are_clipped():
    """The fused reductions and the gathered values see the same clipped rows."""
    arr = get_pileup(_iv([0, 4], [6, 10]), 10)
    lazy = arr[_iv([-3, 8, 12, 2], [2, 15, 20, 2])]
    assert lazy.lengths.cpu().tolist() == [2, 2, 0, 0]
    dense = po.dense_pileup([0, 4], [6, 10], 10)
    assert lazy.tolist() == [dense[0:2].tolist(), dense[8:10].tolist(), [], []]
    assert lazy.sum(axis=-1).cpu().tolist() == [2, 2, 0, 0]
    assert lazy.max(axis=-1).cpu().tolist()[:2] == [1, 1]
    assert lazy.mean(axis=-1).cpu().tolist()[:2] == [1.0, 1.0]
    for how in ("max", "min", "sum"):
        assert torch.equal(getattr(RaggedArray, how)(lazy, axis=-1), getattr(lazy, how)(axis=-1)), how


def test_run_values_are_integers_or_bool():
    arr = get_pileup(_iv([0], [3]), 5)
    with pytest.raises(TypeError):
        arr.astype(float)
    with pytest.raises(TypeError):
        bnp.arithmetics.GenomicRunLengthArray.from_runs([0, 3], [3, 5], [0.5, 1.0])
    assert arr.astype(bool).values.cpu().tolist() == [True, False]


def test_track_indexed_by_a_record_with_left_out_contigs():
    g = bnp.Genome.from_dict({"chr1": 100, "chr1_alt": 50, "chr2": 80}, filter_function=lambda n: "_" not in n)
    track = g.get_intervals(_iv([0, 10], [20, 30], ["chr1", "chr2"])).get_pileup()
    peaks = _iv([5, 0, 15], [25, 10, 25], ["chr1", "chr1_alt", "chr2"])
    with pytest.raises(ValueError, match="leaves out"):
        track[peaks]
    placed = g.get_intervals(peaks)
    assert track[placed].max(axis=-1).cpu().tolist() == [1, 1]
    assert track[_iv([5, 15], [25, 25], ["chr1", "chr2"])].max(axis=-1).cpu().tolist() == [1, 1]
