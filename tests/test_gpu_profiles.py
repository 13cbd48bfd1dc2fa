"""Track profiles on the GPU against tests/profile_oracle.py, bit for bit: the fused column sums of K18 for int64,
bool and float64 tracks (NaN, +-inf, -0.0 and subnormals) at every block and column-tile border, reversed and forward
rows, rows inside one run and rows crossing a run at every position; stranded gathers; locations, windows, clip and
extension; Genome.get_locations; track[locations]; narrowPeak reading; and the summit and TSS profiles of the goldens."""
import gzip
import math
import os

import numpy as np
import pytest
import torch

import bam_oracle as bo
import annotation_oracle as ao
import pileup_oracle as po
import profile_oracle as oracle
import bionumpy_b200 as bnp
from bionumpy_b200 import ops, torch_ops
from bionumpy_b200.arithmetics import FloatRunLengthArray, GenomicRunLengthArray
from bionumpy_b200.arithmetics.intervals import RunsRaggedArray
from bionumpy_b200.io.delimited import NarrowPeakBuffer
from bionumpy_b200.io.exceptions import FormatException

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
TILE = 256                  # the column tile of column_sum_kernel
B = oracle.BLOCK_ROWS
SPECIAL = np.array([math.nan, math.inf, -math.inf, -0.0, 0.0, 5e-324, -2.5e-310, 1e308, -1e308])


def _golden(name):
    return os.path.join(GOLDEN, name)


def bits(values):
    """int64 bit patterns, every NaN as one pattern (NaN equals NaN)."""
    a = np.asarray(values, dtype=np.float64).copy()
    a[np.isnan(a)] = np.nan
    return a.view(np.int64)


def _runs(rng, kind, size, max_run):
    """(run starts int64[R + 1], values) of a random track of ``size`` positions in runs of 1..max_run."""
    lens = rng.integers(1, max_run + 1, size + 1)
    n = int(np.searchsorted(np.cumsum(lens), size)) + 1
    starts = np.minimum(np.concatenate([[0], np.cumsum(lens[:n])]), size).astype(np.int64)
    if kind == "int":
        values = rng.integers(-2 ** 62, 2 ** 62, n, dtype=np.int64)
    elif kind == "bool":
        values = (np.arange(n) + rng.integers(0, 2)) % 2 == 1
    elif kind == "finite":
        values = rng.standard_normal(n) * 1000.0          # moderate magnitudes: every add rounds, nothing saturates
    else:
        values = rng.standard_normal(n) * 10.0 ** rng.integers(-300, 300, n)
        pick = rng.random(n) < 0.1
        values[pick] = SPECIAL[rng.integers(0, SPECIAL.size, int(pick.sum()))]
    return starts, values


def _queries(rng, size, n, width):
    q = rng.integers(0, size - width + 1, n).astype(np.int64)
    q[0] = 0                                   # touches position 0
    q[-1] = size - width                       # touches the last position
    rev = rng.random(n) < 0.5
    return q, rev


SHAPES = [(1, 1), (1, TILE - 1), (B - 1, TILE), (B, TILE + 1), (B + 1, 1), (B + 1, TILE - 1), (3 * B + 17, TILE),
          (600, 2 * TILE + 1), (B + 1, 20011), (3, 20011)]


@pytest.mark.parametrize("kind", ["int", "float"])
@pytest.mark.parametrize("max_run", [1, 7, 10 ** 6])
@pytest.mark.parametrize("n,width", SHAPES)
def test_column_sums_against_the_blocked_oracle(kind, max_run, n, width):
    rng = np.random.default_rng(n * 7919 + width + max_run)
    size = width + 3000
    starts, values = _runs(rng, kind, size, max_run)
    q, rev = _queries(rng, size, n, width)
    want = oracle.column_sum(oracle.rows(oracle.dense(starts, values), q, width, rev))
    ev, q_t = torch.from_numpy(starts).cuda(), torch.from_numpy(q).cuda()
    rev_t = torch.from_numpy(rev.astype(np.uint8)).cuda()
    fn = ops.track_f64_column_sum if kind == "float" else ops.runs_column_sum
    v_t = torch.from_numpy(values).cuda()
    got = fn(ev, v_t, q_t, width, rev_t).cpu().numpy()
    again = fn(ev, v_t, q_t, width, rev_t).cpu().numpy()
    if kind == "float":
        assert np.array_equal(bits(got), bits(want)) and np.array_equal(bits(again), bits(got))
    else:
        assert np.array_equal(got, want) and np.array_equal(again, got)
    forward = fn(ev, v_t, q_t, width).cpu().numpy()
    want_fwd = oracle.column_sum(oracle.rows(oracle.dense(starts, values), q, width))
    assert np.array_equal(bits(forward) if kind == "float" else forward, bits(want_fwd) if kind == "float" else want_fwd)
    # the dispatcher op gives the same
    torch_ops.load()
    name = "track_f64_column_sum" if kind == "float" else "runs_column_sum"
    op = getattr(torch.ops.bnpk, name)(ev, v_t, q_t, width, rev_t).cpu().numpy()
    assert np.array_equal(op.view(np.int64), got.view(np.int64))


def _other_orders(matrix):
    """Column sums of a float matrix in three orders the contract rules out: the block partials folded in reverse
    block order, every row in one pass without blocks, and NumPy's pairwise sum of the transposed matrix."""
    blocks = [oracle.column_sum(matrix[b:b + B]) for b in range(0, matrix.shape[0], B)]
    reverse = np.zeros(matrix.shape[1])
    for p in blocks[::-1]:
        reverse = reverse + p
    one_pass = np.zeros(matrix.shape[1])
    for row in matrix:
        one_pass = one_pass + row
    return {"reverse blocks": reverse, "one pass": one_pass, "pairwise": np.ascontiguousarray(matrix.T).sum(axis=1)}


@pytest.mark.parametrize("max_run", [1, 7])
@pytest.mark.parametrize("n,width", [(B - 1, TILE), (B, TILE + 1), (B + 1, TILE - 1), (3 * B + 17, TILE),
                                     (600, 2 * TILE + 1), (5 * B, 3)])
def test_finite_float_sums_pin_the_summation_order(max_run, n, width):
    """Finite values of moderate size, so every add rounds and no column saturates to inf or NaN: the fixed block
    order is visible in the bits, through the op and through RunsRaggedArray.sum / mean(axis=0)."""
    rng = np.random.default_rng(n * 31 + width + max_run)
    size = width + 2000
    starts, values = _runs(rng, "finite", size, max_run)
    q, rev = _queries(rng, size, n, width)
    matrix = oracle.rows(oracle.dense(starts, values), q, width, rev)
    want = oracle.column_sum(matrix)
    assert np.isfinite(want).all()
    if n <= B:
        assert np.array_equal(bits(want), bits(matrix.sum(axis=0)))        # NumPy's own axis-0 sum
    elif n > B + 1:              # (with one row after the first block every order adds the same two terms)
        for name, other in _other_orders(matrix).items():                  # the data can tell the orders apart
            assert not np.array_equal(bits(other), bits(want)), name
    ev, q_t = torch.from_numpy(starts).cuda(), torch.from_numpy(q).cuda()
    v_t, rev_t = torch.from_numpy(values).cuda(), torch.from_numpy(rev).cuda()
    got = ops.track_f64_column_sum(ev, v_t, q_t, width, rev_t.to(torch.uint8)).cpu().numpy()
    assert np.array_equal(bits(got), bits(want))
    windows = RunsRaggedArray(FloatRunLengthArray(ev, v_t, size), q_t, q_t + width, rev_t)
    assert np.array_equal(bits(windows.sum(axis=0).cpu().numpy()), bits(want))
    assert np.array_equal(bits(windows.mean(axis=0).cpu().numpy()), bits(oracle.column_mean(matrix)))


@pytest.mark.parametrize("kind", ["int", "bool", "float", "finite"])
@pytest.mark.parametrize("n,width", [(1, 5), (B, TILE + 1), (2 * B + 3, 333)])
def test_track_windows_sum_and_mean_axis0(kind, n, width):
    rng = np.random.default_rng(n + width)
    size = width + 1000
    starts, values = _runs(rng, kind, size, 5)
    q, rev = _queries(rng, size, n, width)
    ev = torch.from_numpy(starts).cuda()
    is_float = kind in ("float", "finite")
    if is_float:
        track = FloatRunLengthArray(ev, torch.from_numpy(values).cuda(), size)
    else:
        track = GenomicRunLengthArray(ev, torch.from_numpy(values).cuda(), size)
    q_t = torch.from_numpy(q).cuda()
    windows = RunsRaggedArray(track, q_t, q_t + width, torch.from_numpy(rev).cuda())
    matrix = oracle.rows(oracle.dense(starts, values), q, width, rev)
    s, m = windows.sum(axis=0), windows.mean(axis=0)
    assert s.dtype == (torch.float64 if is_float else torch.int64) and m.dtype == torch.float64
    assert np.array_equal(bits(m.cpu().numpy()), bits(oracle.column_mean(matrix)))
    if is_float:
        assert np.array_equal(bits(s.cpu().numpy()), bits(oracle.column_sum(matrix)))
    else:
        assert np.array_equal(s.cpu().numpy(), oracle.column_sum(matrix))
        # the exact integer sum is the materialised one
        dense_rows = torch.as_tensor(np.asarray(windows)).reshape(n, width).to(torch.int64)
        assert torch.equal(dense_rows.sum(0), s.cpu())
    # the gathered values read reversed rows back to front
    assert np.array_equal(np.asarray(windows).reshape(n, width).view(np.uint8 if kind == "bool" else np.int64),
                          matrix.view(np.uint8 if kind == "bool" else np.int64))


def test_reductions_along_rows_do_not_depend_on_strand():
    rng = np.random.default_rng(5)
    size = 5000
    for kind in ("int", "float"):
        starts, values = _runs(rng, kind, size, 9)
        ev = torch.from_numpy(starts).cuda()
        track = (FloatRunLengthArray if kind == "float" else GenomicRunLengthArray)(ev, torch.from_numpy(values).cuda(),
                                                                                   size)
        a = torch.from_numpy(rng.integers(0, size - 100, 500)).cuda()
        b = a + torch.from_numpy(rng.integers(0, 100, 500)).cuda()
        rev = torch.from_numpy(rng.random(500) < 0.5).cuda()
        plain, flipped = RunsRaggedArray(track, a, b), RunsRaggedArray(track, a, b, rev)
        for how in ("max", "min", "sum", "mean", "any"):
            x = getattr(plain, how)(axis=-1).cpu().numpy()
            y = getattr(flipped, how)(axis=-1).cpu().numpy()
            assert np.array_equal(x.view(np.int64) if x.dtype == np.float64 else x,
                                  y.view(np.int64) if y.dtype == np.float64 else y), how


def test_unequal_and_empty_rows_raise():
    track = GenomicRunLengthArray(torch.tensor([0, 10, 100]).cuda(), torch.tensor([1, 2]).cuda(), 100)
    windows = RunsRaggedArray(track, torch.tensor([0, 5, 9]).cuda(), torch.tensor([10, 15, 20]).cuda())
    for fn in (windows.mean, windows.sum):
        with pytest.raises(NotImplementedError, match=r"^mean\(axis=0\) needs rows of one length: 1 of the 3 rows"):
            fn(axis=0)
    empty = RunsRaggedArray(track, torch.zeros(0, dtype=torch.int64).cuda(), torch.zeros(0, dtype=torch.int64).cuda())
    with pytest.raises(NotImplementedError, match=r"^mean\(axis=0\) needs rows of one length"):
        empty.mean(axis=0)


# --------------------------------------------------------------------------------------------------------------------
# locations, windows, clip and extension
# --------------------------------------------------------------------------------------------------------------------
SIZES = {"a": 100, "b": 50, "c_alt": 30}
ROWS = [("a", 10, 20, "-"), ("a", 10, 20, "+"), ("b", 0, 7, "."), ("a", 95, 100, "-"), ("b", 40, 50, "+"),
        ("a", 0, 3, "-"), ("c_alt", 3, 9, "+")]


def _genome():
    return bnp.Genome.from_dict(SIZES, filter_function=bnp.genomic_data.ignore_underscores)


def _bed6(rows):
    return bnp.Bed6([r[0] for r in rows], [r[1] for r in rows], [r[2] for r in rows], ["x"] * len(rows),
                    [0] * len(rows), "".join(r[3] for r in rows))


def _kept():
    return [r for r in ROWS if "_" not in r[0]]


def _names(text):
    return [text[i].to_string() for i in range(len(text))]


def _strands(strand):
    return "".join("+-."[c] for c in strand.raw().cpu().tolist())


@pytest.mark.parametrize("stranded", [True, False])
@pytest.mark.parametrize("where", ["start", "stop", "center"])
def test_get_location(stranded, where):
    intervals = _genome().get_intervals(_bed6(ROWS), stranded=stranded)
    assert intervals.is_stranded() == stranded and len(intervals) == len(_kept())
    loc = intervals.get_location(where)
    want = [oracle.location(s, e, st if stranded else None, where) for _, s, e, st in _kept()]
    assert loc.position.cpu().tolist() == want
    assert _names(loc.chromosome) == [r[0] for r in _kept()]
    assert loc.is_stranded() == stranded
    data = loc.get_data()
    assert type(data) is (bnp.StrandedLocationEntry if stranded else bnp.LocationEntry)
    if stranded:
        assert _strands(loc.strand) == "".join(r[3] for r in _kept())
    else:
        with pytest.raises(ValueError):
            loc.strand
        with pytest.raises(ValueError):
            intervals.strand


@pytest.mark.parametrize("stranded", [True, False])
@pytest.mark.parametrize("flank,window_size", [(5, None), (0, None), (None, 10), (None, 11), (None, 1), (300, None)])
def test_get_windows_are_clipped_and_keep_the_strand(stranded, flank, window_size):
    genome = _genome()
    loc = genome.get_intervals(_bed6(ROWS), stranded=stranded).get_location("start")
    windows = loc.get_windows(flank=flank, window_size=window_size)
    want = [oracle.window(oracle.location(s, e, st if stranded else None, "start"), SIZES[c], flank, window_size)
            for c, s, e, st in _kept()]
    assert list(zip(windows.start.cpu().tolist(), windows.stop.cpu().tolist())) == want
    assert windows.is_stranded() == stranded
    offsets = {"a": 0, "b": 100}
    assert windows._g_start.cpu().tolist() == [offsets[c] + w[0] for (c, *_), w in zip(_kept(), want)]
    assert windows._g_stop.cpu().tolist() == [offsets[c] + w[1] for (c, *_), w in zip(_kept(), want)]
    # the track read through stranded windows is reversed on '-'
    dense = np.arange(150, dtype=np.int64) * 3
    track = genome.get_track(bnp.BedGraph(["a"] * 100 + ["b"] * 50, list(range(100)) + list(range(50)),
                                          list(range(1, 101)) + list(range(1, 51)), dense.tolist()))
    got = track[windows]
    rows = []
    for (c, s, e, st), (a, b) in zip(_kept(), want):
        row = dense[offsets[c] + a:offsets[c] + b]
        rows.append(row[::-1] if stranded and st == "-" else row)
    assert np.asarray(got).tolist() == np.concatenate(rows).tolist()


def test_window_positions_at_both_contig_ends():
    genome = _genome()
    loc = genome.get_locations(bnp.LocationEntry(["a", "a", "b", "b"], [0, 99, 0, 49]))
    w = loc.get_windows(flank=5)
    assert w.start.cpu().tolist() == [0, 94, 0, 44] and w.stop.cpu().tolist() == [6, 100, 6, 50]


def test_clip_and_extended_to_size():
    genome = _genome()
    for stranded in (True, False):
        iv = genome.get_intervals(_bed6(ROWS), stranded=stranded)
        c = iv.clip()
        assert c.start.cpu().tolist() == [r[1] for r in _kept()] and c.stop.cpu().tolist() == [r[2] for r in _kept()]
        for size in (1, 30, 200):
            ext = iv.extended_to_size(size)
            want = [oracle.extended(s, e, st if stranded else None, size, SIZES[ch]) for ch, s, e, st in _kept()]
            assert list(zip(ext.start.cpu().tolist(), ext.stop.cpu().tolist())) == want
            assert ext.is_stranded() == stranded and type(ext.get_data()) is bnp.Bed6
            pile = np.asarray(ext.get_pileup()["a"])
            dense = po.dense_pileup([w[0] for (ch, *_), w in zip(_kept(), want) if ch == "a"],
                                    [w[1] for (ch, *_), w in zip(_kept(), want) if ch == "a"], 100)
            assert pile.tolist() == dense.tolist()


def test_annotation_features_clip_and_extend_along_their_strand():
    """Transcripts always carry their strand: extended_to_size goes by it and keeps the GTF record type, and the
    result is still read forward when it indexes a track, as the features themselves are."""
    sizes = oracle_sizes(_golden("hg38.chrom.sizes"))
    genome = bnp.Genome.from_file(_golden("hg38.chrom.sizes"))
    transcripts = genome.read_annotation(_golden("gencode_chr21_head.gtf.gz")).transcripts
    rows = ao.select(ao.read(_golden("gencode_chr21_head.gtf.gz"), False), "transcript", False)
    strand = ["+-."[r["strand"]] for r in rows]
    assert set(strand) == {"+", "-"}
    clipped = transcripts.clip()
    assert clipped.start.cpu().tolist() == [r["start"] for r in rows]
    assert clipped.stop.cpu().tolist() == [r["stop"] for r in rows]
    for size in (1, 300, 100_000):
        ext = transcripts.extended_to_size(size)
        want = [oracle.extended(r["start"], r["stop"], st, size, sizes[r["chromosome"].decode()])
                for r, st in zip(rows, strand)]
        assert list(zip(ext.start.cpu().tolist(), ext.stop.cpu().tolist())) == want
        assert type(ext) is type(transcripts) and type(ext.get_data()) is bnp.GFFTranscriptEntry
        assert ext.is_stranded() and _strands(ext.strand) == "".join(strand)
        assert _names(ext.transcript_id) == _names(transcripts.transcript_id)
    pileup = genome.read_intervals(_golden("ctcf_chr21-22_every6th.bam")).get_pileup()
    ext = transcripts.extended_to_size(300)
    dense = _bam_pileups(sizes)["chr21"]
    minus = strand.index("-")
    a, b = ext.start.cpu().tolist()[minus], ext.stop.cpu().tolist()[minus]
    row = pileup[ext[torch.tensor([minus]).cuda()]]
    assert np.asarray(row).tolist() == dense[a:b].tolist()


def test_stranded_flag_through_indexing_sorting_and_merging():
    genome = _genome()
    iv = genome.get_intervals(_bed6(ROWS), stranded=True)
    assert iv[torch.tensor([0, 2]).cuda()].is_stranded()
    assert _strands(iv[[3, 0]].strand) == "--"
    s = iv.sorted()
    assert s.is_stranded() and _strands(s.strand) == "".join(r[3] for r in sorted(_kept(), key=lambda r: r[:3]))
    assert not iv.merged().is_stranded()
    assert not iv[torch.zeros(0, dtype=torch.int64).cuda()].merged().is_stranded()
    with pytest.raises(ValueError):
        genome.get_intervals(bnp.Interval(["a"], [0], [1]), stranded=True)


def test_get_locations_faults_and_track_values():
    genome = _genome()
    with pytest.raises(KeyError):
        genome.get_locations(bnp.LocationEntry(["a", "zz"], [0, 1]))
    for names, pos, row in ((["a", "a"], [0, 100], 1), (["a", "a"], [-1, 3], 0), (["a", "b"], [3, 50], 1)):
        with pytest.raises(ValueError, match=f"location {row} "):
            genome.get_locations(bnp.LocationEntry(names, pos))
    loc = genome.get_locations(bnp.StrandedLocationEntry(["c_alt", "b", "a", "a"], [1, 4, 99, 7], "+-.+"))
    assert len(loc) == 3 and loc.position.cpu().tolist() == [4, 99, 7] and _strands(loc.strand) == "-.+"
    s = loc.sorted()
    assert _names(s.chromosome) == ["a", "a", "b"] and s.position.cpu().tolist() == [7, 99, 4]
    values = np.arange(150) * 0.5 - 3.0
    for dtype in (np.int64, np.float64, np.bool_):
        dense = (values > 0) if dtype == np.bool_ else values.astype(dtype)
        track = genome.get_track(bnp.BedGraph(["a"] * 100 + ["b"] * 50, list(range(100)) + list(range(50)),
                                              list(range(1, 101)) + list(range(1, 51)), dense.tolist()))
        got = track[loc]
        assert got.dtype == track.dtype
        assert got.cpu().numpy().tolist() == dense[[100 + 4, 99, 7]].tolist()


# --------------------------------------------------------------------------------------------------------------------
# narrowPeak
# --------------------------------------------------------------------------------------------------------------------
def _peak_rows(peaks):
    n = len(peaks)
    return list(zip(_names(peaks.chromosome), peaks.start.cpu().tolist(), peaks.stop.cpu().tolist(),
                    _names(peaks.name), peaks.score.cpu().tolist(), _strands(peaks.strand),
                    peaks.signal_value.cpu().tolist(), peaks.p_value.cpu().tolist(), peaks.q_value.cpu().tolist(),
                    peaks.summit.cpu().tolist()))[:n]


@pytest.mark.parametrize("name", ["small_peaks.narrowPeak", "ctcf_chr21-22.bed.gz"])
def test_narrowpeak_reading(name, tmp_path):
    path = _golden(name)
    want = oracle.read_narrowpeak(path)
    kwargs = {} if name.endswith(".narrowPeak") else {"buffer_type": NarrowPeakBuffer}
    peaks = bnp.open(path, **kwargs).read()
    assert type(peaks) is bnp.NarrowPeak and peaks.signal_value.dtype == torch.float64
    assert _peak_rows(peaks) == want
    for size in (300, 5000):
        with bnp.open(path, buffer_type=NarrowPeakBuffer) as f:
            assert sum((_peak_rows(c) for c in f.read_chunks(min_chunk_size=size)), []) == want
    data = gzip.open(path).read() if name.endswith(".gz") else open(path, "rb").read()
    p = str(tmp_path / "x.narrowPeak.gz")
    open(p, "wb").write(gzip.compress(data))
    assert _peak_rows(bnp.open(p).read()) == want


def test_narrowpeak_bad_float_names_its_line():
    good = "chr1\t1\t9\tp\t5\t+\t1.5\t-1\t0.25\t3\n"
    for bad, line in ((good * 2 + good.replace("0.25", "x"), 2), (good.replace("1.5", "nan") + good, 0),
                      (good + "chr1\t1\t9\tp\t5\t+\t1.5\n", 1)):
        with pytest.raises(FormatException) as err:
            NarrowPeakBuffer.from_raw_buffer(bnp.as_encoded_array(bad))
        assert err.value.line_number == line
    buf = NarrowPeakBuffer.from_raw_buffer(bnp.as_encoded_array(good + good[:10]))
    assert _peak_rows(buf.get_data()) == [("chr1", 1, 9, "p", 5, "+", 1.5, -1.0, 0.25, 3)]


# --------------------------------------------------------------------------------------------------------------------
# end to end on the goldens
# --------------------------------------------------------------------------------------------------------------------
def _hg38():
    return oracle_sizes(_golden("hg38.chrom.sizes"))


def oracle_sizes(path):
    return {line.split()[0]: int(line.split()[1]) for line in open(path) if line.strip()}


def _profile(dense, windows, reverse=None):
    m = np.stack([dense[c][a:b] for c, a, b in windows])
    if reverse is not None:
        m[reverse] = m[reverse, ::-1]
    return oracle.column_mean(m)


def _bam_pileups(sizes, strand=None):
    names, _, records, _ = bo.read_bam(_golden("ctcf_chr21-22_every6th.bam"))
    rows = [r for r in bo.bed6_rows(records, names, placed_only=True) if strand is None or r[5] == strand]
    out = {}
    for c in ("chr21", "chr22"):
        mine = [r for r in rows if r[0] == c]
        out[c] = po.dense_pileup([r[1] for r in mine], [r[2] for r in mine], sizes[c])
    return out


def test_summit_profile_of_the_goldens():
    sizes = _hg38()
    genome = bnp.Genome.from_file(_golden("hg38.chrom.sizes"))
    peaks = bnp.open(_golden("ctcf_chr21-22.bed.gz"), buffer_type=NarrowPeakBuffer).read()
    summits = genome.get_locations(bnp.LocationEntry(peaks.chromosome, peaks.start + peaks.summit)).sorted()
    windows = summits.get_windows(flank=200)
    reads = genome.read_intervals(_golden("ctcf_chr21-22_every6th.bam"), stranded=True)
    order = list(sizes)
    want_loc = sorted(((c, s + summit) for c, s, *_, summit in oracle.read_narrowpeak(_golden("ctcf_chr21-22.bed.gz"))),
                      key=lambda x: (order.index(x[0]), x[1]))
    want_windows = [(c,) + oracle.window(p, sizes[c], flank=200) for c, p in want_loc]
    for s in "+-":
        got = reads[reads.strand == s].get_pileup()[windows].mean(axis=0)
        want = _profile(_bam_pileups(sizes, s), want_windows)
        assert got.shape == (401,) and np.array_equal(bits(got.cpu().numpy()), bits(want)), s


def test_tss_profile_of_the_goldens():
    sizes = _hg38()
    genome = bnp.Genome.from_file(_golden("hg38.chrom.sizes"))
    tss = genome.read_annotation(_golden("gencode_chr21_head.gtf.gz")).transcripts.get_location("start")
    assert tss.is_stranded()
    windows = tss.get_windows(flank=500)
    pileup = genome.read_intervals(_golden("ctcf_chr21-22_every6th.bam")).get_pileup()
    got = pileup[windows].mean(axis=0)
    rows = ao.select(ao.read(_golden("gencode_chr21_head.gtf.gz"), False), "transcript", False)
    strand = ["+-."[r["strand"]] for r in rows]
    want_windows = [(r["chromosome"].decode(),) + oracle.window(oracle.location(r["start"], r["stop"], st, "start"),
                                                                sizes[r["chromosome"].decode()], flank=500)
                    for r, st in zip(rows, strand)]
    reverse = np.array([st == "-" for st in strand])
    want = _profile(_bam_pileups(sizes), want_windows, reverse)
    assert got.shape == (1001,) and np.array_equal(bits(got.cpu().numpy()), bits(want))
    # indexing the track with the transcripts themselves stays forward on every strand
    transcripts = genome.read_annotation(_golden("gencode_chr21_head.gtf.gz")).transcripts
    assert pileup[transcripts[torch.tensor([0]).cuda()]].sum(axis=-1).cpu().tolist() == [
        int(_bam_pileups(sizes)["chr21"][rows[0]["start"]:rows[0]["stop"]].sum())]
