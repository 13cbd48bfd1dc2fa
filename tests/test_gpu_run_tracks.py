"""Run-length tracks (GenomicRunLengthArray, the lazy rows of ``track[intervals]`` and GenomicArray) on the GPU against
the dense oracle of tests/pileup_oracle.py: reduce_dense over np.repeat of the runs, never the runs themselves.  Every
value type a track may hold, every query placement that steers the walk of bnpk_runs_reduce and bnpk_runs_extract, and
queries and rows that cross the kernels' grid passes; every fused reduction is also compared with the materialised
reduction of the same rows.

The grid-pass cases size themselves from bnpk_sm_count() and the launch shape of csrc/pileup_kernels.cu:
runs_reduce_kernel and runs_extract_kernel both run sm_count * 8 CTAs of 256 threads with 16 items per thread, so one
pass ("round" in the reduce kernel) covers sm_count * 8 * 256 * 16 (query, run) pairs or output positions."""
import numpy as np
import pytest
import torch

import bionumpy_b200 as bnp
from bionumpy_b200.arithmetics import GenomicRunLengthArray
from bionumpy_b200.genomic_data.genome import GenomicArray
from bionumpy_b200.ragged import RaggedArray

import pileup_oracle as po

pytestmark = pytest.mark.gpu

DTYPES = [np.int64, np.int32, np.int16, np.int8, np.uint8, np.bool_]
HOWS = ("max", "min", "sum", "mean", "any")
CTAS_PER_SM, THREADS, ITEMS = 8, 256, 16       # the launch shape of runs_reduce_kernel and runs_extract_kernel
WARP_ITEMS = 32 * ITEMS


@pytest.fixture(scope="module")
def round_items():
    """(query, run) pairs, or output positions, in one grid pass of the reduce and extract kernels."""
    from bionumpy_b200 import _native as nv
    return int(nv.lib().bnpk_sm_count()) * CTAS_PER_SM * THREADS * ITEMS


def _iv(a, b):
    a, b = np.array(a, dtype=np.int64), np.array(b, dtype=np.int64)
    return bnp.Interval(["chr1"] * a.size, a, b)


def _np(t):
    return t.cpu().numpy() if isinstance(t, torch.Tensor) else np.asarray(t)


def _same(got, want, what=""):
    got, want = _np(got), _np(want)
    assert got.shape == want.shape, what
    if got.dtype.kind == "f" or want.dtype.kind == "f":
        np.testing.assert_array_equal(got.astype(np.float64), want.astype(np.float64), err_msg=str(what))
    else:
        assert got.dtype == want.dtype, (what, got.dtype, want.dtype)
        bad = np.flatnonzero(got != want)
        assert bad.size == 0, (what, bad[:5], got[bad[:5]], want[bad[:5]])


def _wide(rng, dense):
    """int64 values that astype turns into ``dense``: narrow values plus multiples of 2^bits, bools times a nonzero
    factor, changed every 1..3 positions, so runs that differ in int64 become equal neighbours after the cast."""
    blocks = np.repeat(np.arange(dense.size), rng.integers(1, 4, dense.size))[:dense.size]
    k = rng.integers(-3, 4, dense.size + 1)[blocks]
    if dense.dtype == np.bool_:
        return dense.astype(np.int64) * np.where(k == 0, 7, k * 1000 + 1)
    bits = np.dtype(dense.dtype).itemsize * 8
    return dense.astype(np.int64) + (k.astype(np.int64) << bits)


def _track(dense, make="from_runs", rng=None):
    """A track whose values are ``dense``: canonical runs through from_runs, or int64 runs converted by astype (whose
    runs need not be canonical)."""
    if make == "from_runs":
        s, e, v = po.runs_of(dense)
        track = GenomicRunLengthArray.from_runs(s, e, v)
    else:
        wide = _wide(rng, dense)
        s, e, v = po.runs_of(wide)
        track = GenomicRunLengthArray.from_runs(s, e, v).astype(dense.dtype)
        assert track.values.numel() == s.size
    assert track.dtype == torch.from_numpy(np.zeros(0, dense.dtype)).dtype and len(track) == dense.size
    return track


def _rows(dense, a, b):
    """The values of every clipped row, back to back."""
    a, b = po.clip_queries(a, b, dense.size)
    lens = b - a
    first = np.repeat(a - (np.cumsum(lens) - lens), lens)
    return dense[first + np.arange(lens.sum())], lens


def _check_lazy(lazy, dense, a, b, materialise=True):
    """Fused max / min / sum / mean / any of ``lazy`` (the rows [a, b) of a track whose values are ``dense``) against
    the dense oracle, then against the materialised reductions of the same rows, then the rows' values."""
    fused = {}
    for how in HOWS:
        fused[how] = getattr(lazy, how)(axis=-1)
        _same(fused[how], po.reduce_dense(dense, a, b, how), how)
    assert not lazy.is_materialised()
    if not materialise:
        return
    exact = torch.as_tensor(po.mean_is_exact(dense, a, b))
    for how in HOWS:
        mat = getattr(RaggedArray, how)(lazy, axis=-1)
        if how == "mean":
            _same(mat.cpu()[exact], fused[how].cpu()[exact], "materialised mean")
        else:
            _same(mat, fused[how], "materialised " + how)
    values, lens = _rows(dense, a, b)
    _same(lazy.lengths.to(torch.int64), lens, "lengths")
    _same(lazy.ravel(), values, "values")


def _check_rows(track, dense, a, b, materialise=True):
    _check_lazy(track[_iv(a, b)], dense, a, b, materialise)


def _check_whole(track, dense):
    """Whole-track reductions and to_array."""
    for how in HOWS:
        got = getattr(track, how)()
        assert got.dim() == 0
        _same(got.reshape(1), po.reduce_dense(dense, [0], [dense.size], how), "whole " + how)
    _same(track.to_array(), dense, "to_array")


def _random_queries(rng, size, n):
    """Queries reaching past both ends, with reversed, empty, duplicated and nested ones, in random order."""
    a = rng.integers(-5, size + 6, n)
    b = a + rng.integers(-3, size // 3 + 4, n)
    k = n // 8
    a[:k], b[:k] = a[k:2 * k], b[k:2 * k]                                        # duplicated
    a[2 * k:3 * k], b[2 * k:3 * k] = a[3 * k:4 * k] + 1, b[3 * k:4 * k] - 1      # nested
    order = rng.permutation(n)
    return a[order], b[order]


def _empty_queries(size, x):
    """Empty rows of every kind: at a position, reversed, before the track, after it and at its end."""
    return ([x, x + 5, -7, size + 2, size, x + 1], [x, x, -2, size + 9, size, x - 3])


# ---------------------------------------------------------------------------------------------------------------------
# value types
# ---------------------------------------------------------------------------------------------------------------------
MAKES = [(d, "from_runs") for d in DTYPES] + [(d, "astype") for d in DTYPES if d != np.int64]


@pytest.mark.parametrize("dtype,make", MAKES, ids=[f"{np.dtype(d).name}-{m}" for d, m in MAKES])
def test_value_types(dtype, make):
    """Every dtype a track may hold, with its extreme values, made by from_runs and by astype: fused and materialised
    max / min / sum / mean / any over rows that include empty ones, whole-track reductions and to_array."""
    rng = np.random.default_rng(40 + DTYPES.index(dtype))
    size = 4000
    dense = po.random_dense(rng, size, dtype, max_run=6)
    track = _track(dense, make, rng)
    a, b = _random_queries(rng, size, 3000)
    ea, eb = _empty_queries(size, 1234)
    _check_rows(track, dense, np.concatenate([a, ea, [0]]), np.concatenate([b, eb, [size]]))
    _check_whole(track, dense)
    sub = dense[1000:1001]
    _check_whole(track[1000:1001], sub)
    _check_rows(track[1000:1001], sub, [0, 0, -1, 1], [1, 0, 2, 2])


@pytest.mark.parametrize("dtype", DTYPES, ids=[np.dtype(d).name for d in DTYPES])
def test_empty_rows_and_empty_tracks_give_the_dtype_identity(dtype):
    """An empty row's max is the dtype's lowest value and its min the highest (False / True for bool), fused and
    materialised alike; a track of size 0 reduces to the same values."""
    ext = po.extremes(dtype)
    dense = np.repeat(ext, 3)
    track = _track(dense)
    lazy = track[_iv([4, 0, 9, -3, 30], [4, 0, 2, -1, 40])]
    for how in HOWS:
        want = po.reduce_dense(dense, [4, 0, 9, -3, 30], [4, 0, 2, -1, 40], how)
        _same(want, np.full(5, po.empty_value(how, dtype), dtype=want.dtype), how)
        _same(getattr(lazy, how)(axis=-1), want, how)
        if how != "mean":
            _same(getattr(RaggedArray, how)(lazy, axis=-1), want, "materialised " + how)
    for empty in (track[5:5], track[0:0], track[len(track):], track[-1:-4]):
        assert len(empty) == 0
        _check_whole(empty, dense[:0])
        _check_lazy(empty[_iv([0, -2, 1], [0, 3, 0])], dense[:0], [0, -2, 1], [0, 3, 0])


def test_wrapping_sums():
    """Values near +-2^62 over runs of thousands of positions: sums wrap modulo 2^64 (checked against exact Python
    integers too); int32 extremes over millions of positions sum past 2^53 without wrapping."""
    rng = np.random.default_rng(50)
    n_runs = 3000
    lens = rng.integers(500, 3000, n_runs)
    vals = np.where(np.arange(n_runs) % 2 == 0, 1 << 62, -(1 << 62) + (1 << 61)) + rng.integers(0, 1 << 20, n_runs)
    vals[::9] = np.iinfo(np.int64).max - rng.integers(0, 100, vals[::9].size)
    dense = np.repeat(vals.astype(np.int64), lens)
    track = _track(dense)
    size = dense.size
    a = rng.integers(0, size, 200)
    b = a + rng.integers(0, 100_000, 200)
    a, b = np.concatenate([a, [0]]), np.concatenate([b, [size]])
    _check_rows(track, dense, a, b)
    got = track[_iv(a, b)].sum(axis=-1).cpu().numpy()
    ca, cb = po.clip_queries(a, b, size)
    prefix = np.concatenate([[0], np.cumsum(lens)])
    wrapped = 0
    for i in range(0, a.size, 20):
        lo, hi = np.searchsorted(prefix, ca[i], "right") - 1, np.searchsorted(prefix, cb[i], "left")
        cover = np.minimum(prefix[lo + 1:hi + 1], cb[i]) - np.maximum(prefix[lo:hi], ca[i])
        exact = sum(int(v) * int(c) for v, c in zip(vals[lo:hi], cover))
        assert int(got[i]) % 2 ** 64 == exact % 2 ** 64
        wrapped += not -2 ** 63 <= exact < 2 ** 63
    assert wrapped > 0
    _check_whole(track, dense)
    big = np.repeat(np.array([2 ** 31 - 1, -2 ** 31, 2 ** 31 - 1], dtype=np.int32), [3_000_000, 1, 2_000_000])
    t32 = _track(big)
    assert int(t32.sum()) == (2 ** 31 - 1) * 5_000_000 - 2 ** 31 > 2 ** 53
    _check_rows(t32, big, [0, 1, 2_999_999, 3_000_001], [5_000_001, 3_000_001, 3_000_002, 5_000_001])


# ---------------------------------------------------------------------------------------------------------------------
# grid passes
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def big(round_items):
    """A track of 2 rounds + 4096 runs of 1..3 positions, values in [-2^20, 2^20] alternating in sign (so every run
    differs from its neighbours and every sum and mean is exact): (track, dense, run starts, run ends)."""
    rng = np.random.default_rng(60)
    n_runs = 2 * round_items + 4096
    lens = rng.integers(1, 4, n_runs)
    mag = rng.integers(0, 1 << 20, n_runs)
    vals = np.where(np.arange(n_runs) % 2 == 0, mag + 1, -mag)
    ends = np.cumsum(lens)
    starts = ends - lens
    track = GenomicRunLengthArray.from_runs(starts, ends, vals)
    return track, np.repeat(vals, lens), starts, ends


def _over_runs(starts, ends, first, counts):
    """Queries over ``counts[i]`` consecutive runs each, back to back from run ``first`` (a count of 0 is an empty
    query at the next run's start)."""
    a, b, r = [], [], first
    for c in counts:
        a.append(starts[r])
        b.append(ends[r + c - 1] if c else starts[r])
        r += c
    return np.array(a), np.array(b)


@pytest.mark.parametrize("runs", ["round-1", "round", "round+1", "2round+5"])
def test_one_query_across_grid_passes(big, round_items, runs):
    """One query over round - 1, round, round + 1 and 2 rounds + 5 runs: the reduce walk takes one, one, two and three
    passes, and the materialised row spans several extract passes."""
    track, dense, starts, ends = big
    n = {"round-1": round_items - 1, "round": round_items, "round+1": round_items + 1,
         "2round+5": 2 * round_items + 5}[runs]
    a, b = _over_runs(starts, ends, 3, [n])
    _check_rows(track, dense, np.concatenate([a, a + 1]), np.concatenate([b, b - 1]))


@pytest.mark.parametrize("lead", [5, 16, WARP_ITEMS, WARP_ITEMS + 3])
def test_query_that_begins_just_before_the_round_border(big, round_items, lead):
    """The second query begins ``lead`` pairs before the first round border: the last warp of round 0 holds two
    queries (or, for a whole warp's lead, only the second), and the first warp of round 1 lies wholly inside it."""
    track, dense, starts, ends = big
    a, b = _over_runs(starts, ends, 0, [round_items - lead, lead + 3 * WARP_ITEMS + 7, 100, 2])
    _check_rows(track, dense, a, b)


@pytest.mark.parametrize("shift", [0, 2, 9])
def test_round_border_among_short_queries(big, round_items, shift):
    """Queries of 7 runs, with empty queries between some of them, around the first round border: the border falls
    inside one of them or, for shift 2, exactly between two."""
    track, dense, starts, ends = big
    counts = [round_items - 100 + shift]
    for i in range(40):
        counts += [7, 0] if i % 3 == 0 else [7]
    counts.append(1000)
    a, b = _over_runs(starts, ends, 0, counts)
    _check_rows(track, dense, a, b)


def test_extract_across_grid_passes(big, round_items):
    """to_array of a track more than 3 extract passes long, and a slice and position list that cross the passes."""
    track, dense, starts, ends = big
    assert dense.size > 3 * round_items
    _same(track.to_array(), dense, "to_array")
    lo, hi = round_items - 3, 2 * round_items + 7
    sub = track[lo:hi]
    _same(sub.to_array(), dense[lo:hi], "slice")
    s, e, v = po.runs_of(dense[lo:hi])
    _same(sub.starts, s, "slice starts")
    _same(sub.ends, e, "slice ends")
    _same(sub.values, v, "slice values")
    pos = np.random.default_rng(61).integers(0, dense.size, round_items + 1000)
    _same(track[torch.as_tensor(pos)], dense[pos], "positions")


# ---------------------------------------------------------------------------------------------------------------------
# query placement
# ---------------------------------------------------------------------------------------------------------------------
def _placement_track(run_len, dtype=np.int64, n_runs=3000, seed=70):
    """A track of about ``n_runs`` runs of 1..run_len positions; with run_len 1 (int64 only) every run is one
    position long: neighbouring values differ in their lowest bit."""
    rng = np.random.default_rng(seed)
    dense = po.random_dense(rng, n_runs * (1 if run_len == 1 else 2), dtype, max_run=run_len)
    if run_len == 1:
        dense = (dense & ~np.int64(1)) | (np.arange(dense.size) & 1)
        assert po.runs_of(dense)[0].size == dense.size
    return _track(dense), dense


@pytest.mark.parametrize("run_len", [1, 3])
def test_query_border_at_every_chunk_offset(run_len):
    """A first query of 0..31 runs puts the next border at every offset of a 16-item work chunk, and queries of 1..33
    runs follow; with runs of one position the extract chunks see the same borders."""
    track, dense = _placement_track(run_len)
    s, e, _ = po.runs_of(dense)
    for lead in range(32):
        a, b = _over_runs(s, e, 0, [lead] + list(range(1, 34)) + [1, 0, 1])
        _check_rows(track, dense, a, b, materialise=lead % 4 == 0 or lead == 31)


@pytest.mark.parametrize("n_empty", [1, 2, 20])
def test_empty_queries_inside_one_chunk(n_empty):
    """Runs of 1, 2 and 20 empty queries of every kind between non-empty queries inside one work chunk, at every
    offset of the chunk."""
    track, dense = _placement_track(1, n_runs=400)
    size = dense.size
    for lead in range(16):
        qa, qb = [0, lead], [lead, lead + 3]
        for x, n_next in ((lead + 3, 4), (lead + 7, 30)):
            ea, eb = _empty_queries(size, x + 1)
            reps = -(-n_empty // len(ea))
            qa += (ea * reps)[:n_empty] + [x]
            qb += (eb * reps)[:n_empty] + [x + n_next]
        ea, eb = _empty_queries(size, 50)
        qa, qb = qa + (ea * 4)[:n_empty], qb + (eb * 4)[:n_empty]
        _check_rows(track, dense, qa, qb)


@pytest.mark.parametrize("dtype", [np.int64, np.int8, np.bool_], ids=["int64", "int8", "bool"])
def test_borders_at_run_starts(dtype):
    """Every pair of points among 0, 1, size - 1, size, each run start -1 / 0 / +1 and points outside the track: all
    placements of both borders on and next to runs, reversed, empty, nested and duplicated queries."""
    track, dense = _placement_track(6, dtype, n_runs=12, seed=71)
    size = dense.size
    s, _, _ = po.runs_of(dense)
    pts = np.unique(np.concatenate([[0, 1, size - 1, size, -3, size + 2], s - 1, s, s + 1]))
    a, b = np.repeat(pts, pts.size), np.tile(pts, pts.size)
    _check_rows(track, dense, a, b)
    _check_rows(track, dense, a[::-1], b[::-1], materialise=False)


@pytest.mark.parametrize("dtype", DTYPES, ids=[np.dtype(d).name for d in DTYPES])
def test_reversed_outside_duplicated_nested_unsorted_queries(dtype):
    rng = np.random.default_rng(72)
    track, dense = _placement_track(5, dtype, n_runs=2000, seed=72)
    size = dense.size
    a, b = _random_queries(rng, size, 5000)
    a = np.concatenate([a, [-10, -10, size - 1, size + 1, 7, 3, 3, 0], [10, 12, 11]])
    b = np.concatenate([b, [-1, 5, size + 10, size + 4, 3, 3, 3, size], [20, 18, 19]])
    _check_rows(track, dense, a, b)


@pytest.mark.parametrize("dtype", DTYPES, ids=[np.dtype(d).name for d in DTYPES])
def test_one_run_and_size_one_tracks(dtype):
    ext = po.extremes(dtype)
    for dense in (np.full(50, ext[0]), np.full(50, ext[-1]), ext[:1], ext[-1:]):
        track = _track(dense)
        assert track.values.numel() == 1
        pts = np.arange(-2, dense.size + 3)
        pts = pts[(pts < 3) | (pts > dense.size - 3)]
        _check_rows(track, dense, np.repeat(pts, pts.size), np.tile(pts, pts.size))
        _check_whole(track, dense)


# ---------------------------------------------------------------------------------------------------------------------
# indexing
# ---------------------------------------------------------------------------------------------------------------------
def _check_slice(track, dense, a, b):
    sub = track[a:b]
    want = dense[a:b]
    assert len(sub) == want.size, (a, b)
    _same(sub.to_array(), want, (a, b))
    if want.size:
        s, e, v = po.runs_of(want)
        _same(sub.starts, s, (a, b, "starts"))
        _same(sub.ends, e, (a, b, "ends"))
        _same(sub.values, v, (a, b, "values"))
    return sub, want


@pytest.mark.parametrize("dtype", DTYPES, ids=[np.dtype(d).name for d in DTYPES])
def test_indexing(dtype):
    """arr[int] (negative too), arr[list | ndarray | tensor], and arr[a:b] with a == b, bounds on run borders -1 / 0
    / +1, negative bounds and bounds past the end, against the dense slice."""
    rng = np.random.default_rng(80)
    dense = po.random_dense(rng, 300, dtype, max_run=9)
    track = _track(dense)
    size = dense.size
    s, _, _ = po.runs_of(dense)
    border = int(s[len(s) // 2])
    for i in [0, 1, size - 1, -1, -size, border - 1, border, border + 1, np.int64(5), np.int32(-2)]:
        assert track[i] == dense[i].item(), i
    for i in (size, -size - 1):
        with pytest.raises(IndexError):
            track[i]
    pos = rng.integers(0, size, 500)
    for idx in (pos.tolist(), pos, torch.as_tensor(pos), torch.as_tensor(pos).cuda(), pos[:0], [border]):
        _same(track[idx], dense[np.asarray(idx.cpu() if isinstance(idx, torch.Tensor) else idx, dtype=np.int64)],
              type(idx))
    with pytest.raises(IndexError):
        track[[0, size]]
    with pytest.raises(IndexError):
        track[np.array([-1])]
    bounds = [None, 0, 1, border - 1, border, border + 1, size - 1, size, size + 5, -1, -3, -size, -size - 4]
    for a in bounds:
        for b in bounds:
            _check_slice(track, dense, a, b)
    sub, want = _check_slice(track, dense, border - 1, size - 2)
    _check_whole(sub, want)
    _check_rows(sub, want, [0, 1, 5, -1, 0], [want.size, 1, 2, 3, want.size + 4])
    sub2, want2 = _check_slice(sub, want, 1, -1)
    _check_whole(sub2, want2)


# ---------------------------------------------------------------------------------------------------------------------
# genome tracks
# ---------------------------------------------------------------------------------------------------------------------
SIZES = {"one": 1, "a": 37, "alt_x": 9, "two": 1, "b": 50, "none": 20, "c": 64, "d": 30, "last": 1}


def _genome():
    return bnp.Genome.from_dict(SIZES, filter_function=lambda n: "_" not in n)


def _check_genome_track(track, dense, names, offsets):
    assert list(track.to_dict()) == names
    for name, arr in track.to_dict().items():
        off, size = offsets[name], SIZES[name]
        want = dense[off:off + size]
        for got in (arr, track[name]):
            assert len(got) == size, name
            s, e, v = po.runs_of(want)
            _same(got.starts, s, name)
            _same(got.ends, e, name)
            _same(got.values, v, name)
            _same(got.to_array(), want, name)
        _check_whole(track[name], want)


def _genome_queries(rng, names, offsets):
    """Per included contig: the whole contig, empty rows at both ends, single positions and random rows."""
    chroms, a, b = [], [], []
    for name in names:
        size = SIZES[name]
        rows = [(0, size), (0, 0), (size, size), (0, 1), (size - 1, size)]
        for _ in range(6):
            x = int(rng.integers(0, size + 1))
            rows.append((x, int(rng.integers(x, size + 1))))
        for s, e in rows:
            chroms.append(name)
            a.append(s)
            b.append(e)
    a, b = np.array(a), np.array(b)
    g0 = np.array([offsets[c] for c in chroms])
    return chroms, a, b, g0 + a, g0 + b


def test_genome_pileup_contigs_and_rows():
    """A pileup over contigs of size 1, a left-out contig and contigs with no interval: track[name], to_dict() and
    track[intervals] reductions across contigs against dense per-contig slices."""
    rng = np.random.default_rng(90)
    g = _genome()
    names, offsets, total = po.genome_layout(SIZES)
    assert "alt_x" not in names and total == sum(SIZES.values()) - SIZES["alt_x"]
    chroms = ["a", "a", "one", "b", "b", "c", "c", "c", "last", "alt_x", "b"]
    starts = np.array([0, 30, 0, 10, 49, 0, 5, 63, 0, 2, 0])
    stops = np.array([37, 37, 1, 20, 50, 64, 60, 64, 1, 7, 50])
    placed = g.get_intervals(bnp.Interval(chroms, starts, stops))
    _, gs, ge = po.genome_intervals(SIZES, chroms, starts, stops)
    qc, qa, qb, qga, qgb = _genome_queries(rng, names, offsets)
    peaks = g.get_intervals(bnp.Interval(qc, qa, qb))
    for track, dense in ((placed.get_pileup(), po.dense_pileup(gs, ge, total)),
                         (placed.get_mask(), po.dense_pileup(gs, ge, total) > 0)):
        _check_genome_track(track, dense, names, offsets)
        _check_lazy(track[peaks], dense, qga, qgb)
        _check_lazy(track[bnp.Interval(qc, qa, qb)], dense, qga, qgb, materialise=False)


@pytest.mark.parametrize("dtype", [np.int64, np.int16, np.bool_], ids=["int64", "int16", "bool"])
def test_genome_track_of_any_runs(dtype):
    """A genome track from runs whose borders do and do not fall on contig borders, a run that spans three contigs
    and contigs of size 1 inside a run: every contig and row against the dense array."""
    rng = np.random.default_rng(91)
    g = _genome()
    names, offsets, total = po.genome_layout(SIZES)
    dense = po.random_dense(rng, total, dtype, max_run=8)
    ext = po.extremes(dtype)
    b0, c0 = offsets["b"], offsets["c"]
    dense[:b0] = ext[-1]                                         # "one", "a" and "two" in one run
    dense[b0] = ext[0]                                           # a run border on the contig border of "b"
    dense[c0 - 1] = dense[c0] = ext[0]                           # no run border on the contig border of "c"
    dense[offsets["last"]] = dense[offsets["last"] - 1]          # the last contig inside the run before it
    s, e, v = po.runs_of(dense)
    track = GenomicArray(torch.as_tensor(np.append(s, total)).cuda(), torch.as_tensor(v).cuda(), g)
    _check_genome_track(track, dense, names, offsets)
    qc, qa, qb, qga, qgb = _genome_queries(rng, names, offsets)
    _check_lazy(track[g.get_intervals(bnp.Interval(qc, qa, qb))], dense, qga, qgb)
