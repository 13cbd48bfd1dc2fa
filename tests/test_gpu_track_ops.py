"""Track operators and interval intersections on the GPU at the places where runs_combine_kernel and
interval_intersect_kernel split their work, against oracles that never look at the runs under test: dense NumPy arrays
(po.dense_of of the input runs, so.dense_op, po.runs_of for the canonical runs, po.reduce_dense) and plain Python
loops (so.sweep_loop, so.sort_intervals).

Geometry of both kernels (csrc/pileup_kernels.cu): 256 threads x 8 items = 2048 merged run starts (or rows) per tile.
so.event_tracks places a chosen run start, or an A/B tie, at a chosen merged index and asserts the placement, so the
cases below put changes on thread borders (merged index = 0 mod 8) and tile borders (= 0 mod 2048)."""
import warnings
from fractions import Fraction

import numpy as np
import pytest
import torch

import bionumpy_b200 as bnp
from bionumpy_b200 import _native as nv
from bionumpy_b200 import ops
from bionumpy_b200.arithmetics import (GenomicRunLengthArray, count_overlap, forbes, get_boolean_mask,
                                       global_intersect, intersect, jaccard, sort_intervals)
from bionumpy_b200.arithmetics.intervals import NAME_BYTES, NAME_SLOTS
from bionumpy_b200.genomic_data.genome import GenomicArray

import interval_sets_oracle as so
import pileup_oracle as po

pytestmark = pytest.mark.gpu

TILE, ITEMS = 2048, 8
OPS = [np.add, np.subtract, np.multiply, np.bitwise_and, np.bitwise_or, np.bitwise_xor, np.minimum, np.maximum,
       np.equal, np.not_equal, np.less, np.less_equal, np.greater, np.greater_equal]
LOGICAL = [np.logical_and, np.logical_or, np.logical_xor]
TYPES = [np.int8, np.int16, np.int32, np.uint8, np.int64, np.bool_]


def _launches(fn):
    lib = nv.load_library()
    torch.cuda.synchronize()
    before = lib.bnpk_launch_count()
    out = fn()
    torch.cuda.synchronize()
    return out, lib.bnpk_launch_count() - before


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


def _track(runs):
    s, e, v = runs
    return GenomicRunLengthArray.from_runs(s, e, torch.from_numpy(np.asarray(v)))


def _check(got, want, what=""):
    """The runs, values, dtype and length of ``got`` against the canonical runs of the dense ``want``."""
    s, e, v = po.runs_of(want)
    assert isinstance(got, GenomicRunLengthArray), what
    assert len(got) == want.size, what
    assert got.dtype == torch.from_numpy(want[:0]).dtype, (what, got.dtype, want.dtype)
    for name, g, w in (("starts", got.starts, s), ("ends", got.ends, e), ("values", got.values, v)):
        g = g.cpu().numpy()
        assert g.shape == w.shape and np.array_equal(g, w), (what, name, np.flatnonzero(g != w)[:5] if
                                                            g.shape == w.shape else (g.shape, w.shape))


def _expect(ufunc, x, y, dx, dy, what=""):
    """ufunc(x, y) on tracks or scalars against the same ufunc on the dense operands; an operation NumPy refuses must
    raise the exception NumPy raises."""
    try:
        want = so.dense_op(ufunc, dx, dy)[0]
    except Exception as e:      # noqa: BLE001 -- the exception type is the expectation
        with pytest.raises(type(e)):
            ufunc(x, y)
        return
    if want.dtype.kind == "f" or (want.dtype.kind == "u" and want.dtype.itemsize > 1):
        # float, uint16, uint32 and uint64 results take the dense path: NumPy's own answer on the tracks' dense
        # arrays in their own dtypes (a uint8 track + np.uint64(5) is uint64 there, not the float64 of int64 + uint64)
        with np.errstate(over="ignore"):
            want = ufunc(dx, dy)
        got = ufunc(x, y)
        assert isinstance(got, np.ndarray) and got.dtype == want.dtype and np.array_equal(got, want), what
        return
    _check(ufunc(x, y), want, what)


# --------------------------------------------------------------------------------------------------------------------
# combine at the merge-path splits
# --------------------------------------------------------------------------------------------------------------------
SPLITS = [8, 16, 2040, 2047, 2048, 2049, 2056, 4096, 2048 * 40]
# (A before, B before, A after, B after) around the placed event; a side that starts no run keeps its value
CHANGES = {
    "only_a": (1, 2, 5, 2),
    "only_b": (1, 2, 1, 6),
    "both": (1, 2, 4, 7),
    "plus_cancels": (3, 5, 4, 4),          # A + 1, B - 1: + and == of the result do not change
    "masked_by_zero": (6, 0, 3, 0),        # &, * and min with 0 do not change
    "zero_both": (6, 0, 0, 3),             # both change, & and * stay 0
    "swapped": (9, 2, 2, 9),               # both change, + * & | ^ min max != stay
    "masked_by_max": (1, 5, 2, 5),         # max and | stay
    "equal_neighbours": (4, 4, 4, 4),      # both start a run with the value they had
    "astype_equal": (1, 2, 257, 2),        # 1 -> 257: equal after astype(bool) and astype(int8)
}
# the placed event and where its first merged start goes: an A start at m, a B start at m, a tie at (m - 1, m) and
# a tie at (m, m + 1)
PLACEMENTS = {"a_at_m": ("a", 0), "b_at_m": ("b", 0), "tie_m-1_m": ("ab", -1), "tie_m_m+1": ("ab", 0)}
CAST_CHANGES = ("only_a", "both", "equal_neighbours", "astype_equal")


def _casts(a, b, da, db, change):
    yield "int64", _track(a), _track(b), da, db
    if change in CAST_CHANGES:
        yield "bool", _track(a).astype(bool), _track(b).astype(bool), da != 0, db != 0
        yield "int8", _track(a).astype(np.int8), _track(b).astype(np.int8), da.astype(np.int8), db.astype(np.int8)


def _run_layout(a, b, label, ops_=OPS, casts=True, change="only_a"):
    da, db = po.dense_of(*a), po.dense_of(*b)
    for cast, x, y, dx, dy in (_casts(a, b, da, db, change) if casts else [("int64", _track(a), _track(b), da, db)]):
        for ufunc in ops_:
            _expect(ufunc, x, y, dx, dy, (label, cast, ufunc.__name__))


@pytest.mark.parametrize("m", SPLITS)
def test_combine_change_at_split(m):
    """Every change of CHANGES, as an A start, a B start or a tie, at merged index m (and the tie at m - 1 / m):
    the thread or tile that holds m decides alone whether a run begins there."""
    for place, (side, shift) in PLACEMENTS.items():
        for change, (a0, b0, a1, b1) in CHANGES.items():
            # the "ab" set-up event fixes the values just before the placed one
            a, b, _, _ = so.event_tracks([("ab", a0, b0), (side, a1, b1)], 1, m + shift, after=21, seed=m)
            _run_layout(a, b, (m, place, change), change=change)


@pytest.mark.parametrize("k", [2, 8, 9, 2048])
@pytest.mark.parametrize("m", [2040, 2047, 2048])
def test_combine_consecutive_ties(k, m):
    """k ties in a row from merged index m; with k = 2048 from m = 2048 the whole second tile is ties."""
    vals = [((i * 7) % 3, (i * 5) % 4) for i in range(k)]          # masked, equal and changing pairs mixed
    a, b, _, _ = so.event_tracks([("ab", x, y) for x, y in vals], 0, m, after=13, seed=k + m)
    _run_layout(a, b, (k, m), casts=k < 2048)


@pytest.mark.parametrize("total", [2 * TILE + 1, 2 * TILE + ITEMS, TILE + 1, TILE + ITEMS])
@pytest.mark.parametrize("side", ["a", "b", "ab"])
def test_combine_last_tile(total, side):
    """The last tile holds 1 or 8 merged starts, the last of them the placed event."""
    m = total - (2 if side == "ab" else 1)
    for change in ("only_a", "both", "equal_neighbours", "masked_by_zero"):
        a0, b0, a1, b1 = CHANGES[change]
        a, b, _, _ = so.event_tracks([("ab", a0, b0), (side, a1, b1)], 1, m, after=0, seed=total)
        assert a[0].size + b[0].size == total
        _run_layout(a, b, (total, side, change), casts=False)


def test_combine_size_one_tracks():
    for dx in (np.int64, np.bool_, np.int8):
        for dy in (np.int64, np.bool_, np.uint8):
            for vx in po.extremes(dx):
                for vy in po.extremes(dy)[:3]:
                    x = GenomicRunLengthArray.from_runs([0], [1], torch.from_numpy(np.array([vx])))
                    y = GenomicRunLengthArray.from_runs([0], [1], torch.from_numpy(np.array([vy])))
                    for ufunc in OPS:
                        _expect(ufunc, x, y, np.array([vx]), np.array([vy]), (dx, dy, vx, vy))


def test_combine_one_run_against_unit_runs():
    rng = np.random.default_rng(3)
    size = 3 * TILE + 5
    one = (np.array([0]), np.array([size]), np.array([2]))
    unit = (np.arange(size), np.arange(1, size + 1), rng.integers(-3, 4, size))     # equal neighbours too
    _run_layout(one, unit, "one_vs_unit", casts=False)
    _run_layout(unit, one, "unit_vs_one", casts=False)


# --------------------------------------------------------------------------------------------------------------------
# operand types
# --------------------------------------------------------------------------------------------------------------------
def _typed(rng, dtype, size, how):
    """(track, dense) of ``dtype`` holding its extremes, made by from_runs or by astype of wider int64 runs that the
    cast maps onto the same values (so neighbouring runs may be equal)."""
    dense = po.random_dense(rng, size, dtype, max_run=3)
    ext = po.extremes(dtype)
    dense[:ext.size] = ext
    if how == "from_runs":
        return _track(po.runs_of(dense)), dense
    if dtype == np.bool_:
        wide = dense.astype(np.int64) * rng.choice([1, 2, -5, 1 << 40], size)
    elif dtype == np.int64:
        wide = dense
    else:
        bits = np.iinfo(dtype).bits
        wide = dense.astype(np.int64) + rng.integers(-3, 4, size) * (1 << bits)
    return _track(po.runs_of(wide)).astype(dtype), dense


@pytest.mark.parametrize("ty", TYPES, ids=lambda t: np.dtype(t).name)
@pytest.mark.parametrize("tx", TYPES, ids=lambda t: np.dtype(t).name)
def test_operand_type_pairs(tx, ty):
    rng = np.random.default_rng(TYPES.index(tx) * 10 + TYPES.index(ty))
    for hx, hy in (("from_runs", "astype"), ("astype", "from_runs")):
        x, dx = _typed(rng, tx, 700, hx)
        y, dy = _typed(rng, ty, 700, hy)
        for ufunc in OPS + LOGICAL:
            _expect(ufunc, x, y, dx, dy, (hx, hy, ufunc.__name__))


SCALARS = [0, 1, -1, 2 ** 63 - 1, -2 ** 63, 2 ** 63, True, False, np.int8(-128), np.int8(127), np.int16(-32768),
           np.int32(2 ** 31 - 1), np.int64(-2 ** 63), np.uint8(255), np.bool_(True), np.bool_(False),
           np.uint16(65535), np.uint32(2 ** 32 - 1), np.uint64(5), np.uint64(2 ** 64 - 1)]


@pytest.mark.parametrize("how", ["from_runs", "astype"])
@pytest.mark.parametrize("tx", TYPES, ids=lambda t: np.dtype(t).name)
def test_scalar_operands(tx, how):
    """Python and NumPy scalars on either side; the result dtype is NumPy's on the dense operands (integer tracks
    computed as int64; float, uint16, uint32 and uint64 results are NumPy's dense arrays), and what NumPy refuses
    raises its exception."""
    rng = np.random.default_rng(TYPES.index(tx))
    x, dx = _typed(rng, tx, 300, how)
    for s in SCALARS:
        for ufunc in OPS + LOGICAL:
            _expect(ufunc, x, s, dx, s, (repr(s), ufunc.__name__))
            _expect(ufunc, s, x, s, dx, (repr(s), ufunc.__name__, "reflected"))


@pytest.mark.parametrize("tx", TYPES, ids=lambda t: np.dtype(t).name)
def test_unary_operators(tx):
    rng = np.random.default_rng(40 + TYPES.index(tx))
    for how in ("from_runs", "astype"):
        x, dx = _typed(rng, tx, 500, how)
        wide = so.widen(dx)
        _check(~x, ~wide, (how, "~"))
        _check(np.invert(x), ~wide, (how, "invert"))
        _check(np.logical_not(x), np.logical_not(dx), (how, "logical_not"))
        if tx == np.bool_:
            with pytest.raises(TypeError):
                -x
        else:
            with np.errstate(over="ignore"):
                _check(-x, -wide, (how, "-"))


# --------------------------------------------------------------------------------------------------------------------
# GenomicArray
# --------------------------------------------------------------------------------------------------------------------
SIZES = {"one": 1, "a": 37, "alt_x": 9, "two": 1, "b": 50, "none": 20, "c": 64, "d": 30, "last": 1}


def _genome(sizes=SIZES):
    return bnp.Genome.from_dict(sizes, filter_function=lambda n: "_" not in n)


def _check_genome(track, dense, names, offsets, what):
    assert isinstance(track, GenomicArray), what
    _check(track._global, dense, what)
    for name, arr in track.to_dict().items():
        want = dense[offsets[name]:offsets[name] + SIZES[name]]
        _check(arr, want, (what, name, "to_dict"))
        _check(track[name], want, (what, name))
    assert list(track.to_dict()) == names


def test_genomic_array_operators_per_contig():
    rng = np.random.default_rng(50)
    g = _genome()
    names, offsets, total = po.genome_layout(SIZES)
    chroms = ["a", "a", "one", "b", "b", "c", "c", "c", "last", "alt_x", "b", "d"]
    starts = np.array([0, 30, 0, 10, 49, 0, 5, 63, 0, 2, 0, 29])
    stops = np.array([37, 37, 1, 20, 50, 64, 60, 64, 1, 7, 50, 30])
    _, gs, ge = po.genome_intervals(SIZES, chroms, starts, stops)
    pileup = g.get_intervals(bnp.Interval(chroms, starts, stops)).get_pileup()
    dp = po.dense_pileup(gs, ge, total)
    mchroms = ["one", "two", "a", "b", "c", "alt_x", "last"]
    ms, me = np.array([0, 0, 36, 0, 63, 0, 0]), np.array([1, 1, 37, 25, 64, 9, 1])
    _, mgs, mge = po.genome_intervals(SIZES, mchroms, ms, me)
    mask = g.get_intervals(bnp.Interval(mchroms, ms, me)).get_mask()
    dm = po.dense_mask(mgs, mge, total)
    mask2 = g.get_intervals(bnp.Interval(chroms, starts, stops)).get_mask()
    dm2 = dp > 0
    cases = [("pileup&mask", pileup & mask, dp & dm), ("mask*pileup", mask * pileup, dm * dp),
             ("pileup+mask", pileup + mask, dp + dm), ("pileup-3", pileup - 3, dp - 3),
             ("2*pileup", 2 * pileup, 2 * dp), ("pileup>1", pileup > 1, dp > 1), ("pileup==0", pileup == 0, dp == 0),
             ("mask&mask", mask & mask2, dm & dm2), ("mask|mask", mask | mask2, dm | dm2),
             ("mask^mask", mask ^ mask2, dm ^ dm2), ("mask==mask", mask == mask2, dm == dm2),
             ("mask<mask", mask < mask2, dm < dm2), ("pileup>=mask", pileup >= mask, dp >= dm),
             ("~mask", ~mask, ~dm), ("-pileup", -pileup, -dp),
             ("max", np.maximum(pileup, mask), np.maximum(dp, dm)), ("min", np.minimum(pileup, 1), np.minimum(dp, 1)),
             ("logical_and", np.logical_and(pileup, mask), np.logical_and(dp, dm)), ("mask&True", mask & True, dm)]
    qc, qa, qb = [], [], []
    for name in names:
        size = SIZES[name]
        for s, e in [(0, size), (0, 0), (size, size), (0, 1), (size - 1, size)] + \
                [tuple(sorted(rng.integers(0, size + 1, 2))) for _ in range(4)]:
            qc.append(name)
            qa.append(int(s))
            qb.append(int(e))
    qa, qb = np.array(qa), np.array(qb)
    g0 = np.array([offsets[c] for c in qc])
    peaks = g.get_intervals(bnp.Interval(qc, qa, qb))
    for what, got, want in cases:
        _check_genome(got, want, names, offsets, what)
        rows = got[peaks]
        mx = rows.max(axis=-1).cpu().numpy()
        assert np.array_equal(mx, po.reduce_dense(want, g0 + qa, g0 + qb, "max")), what
        assert mx.dtype == want.dtype, what
        assert np.array_equal(rows.sum(axis=-1).cpu().numpy(), po.reduce_dense(want, g0 + qa, g0 + qb, "sum")), what


def test_genomic_array_other_genome_raises():
    g = _genome()
    t = g.get_intervals(bnp.Interval(["a"], [1], [5])).get_mask()
    other_size = dict(SIZES, d=31)
    other_order = dict(reversed(list(SIZES.items())))
    for sizes in (other_size, other_order):
        u = _genome(sizes).get_intervals(bnp.Interval(["a"], [1], [5])).get_mask()
        with pytest.raises(ValueError):
            t & u
        with pytest.raises(ValueError):
            np.maximum(u, t)


# --------------------------------------------------------------------------------------------------------------------
# bnpk_interval_intersect directly
# --------------------------------------------------------------------------------------------------------------------
def _dev(x, dtype=torch.int64):
    return torch.as_tensor(np.asarray(x)).to("cuda", dtype)


def _sweep(start, stop, same=None, what=""):
    """Both forms of bnpk_interval_intersect against so.sweep_loop, one launch each."""
    rows_want, stops_want, over_want = so.sweep_loop(start, stop, same)
    st, sp = _dev(start), _dev(stop)
    sm = None if same is None else _dev(same, torch.uint8)
    (rows, stops, n_out, over), launches = _launches(lambda: ops.interval_intersect(st, sp, sm, rows=True))
    k = int(n_out.item())
    assert launches == (1 if len(start) else 0), what
    assert k == rows_want.size, (what, k, rows_want.size)
    assert np.array_equal(rows[:k].cpu().numpy(), rows_want), what
    assert np.array_equal(stops[:k].cpu().numpy(), stops_want), what
    assert int(over.item()) == over_want, what
    (r2, s2, n2, o2), launches = _launches(lambda: ops.interval_intersect(st, sp, sm, rows=False))
    assert r2 is None and s2 is None and launches == (1 if len(start) else 0), what
    assert int(n2.item()) == k and int(o2.item()) == over_want, what


def _no_pairs(n):
    start = 4 * np.arange(n, dtype=np.int64)
    return start, start + 2           # stop[i - 1] = 4 i - 2 < start[i]


@pytest.mark.parametrize("m", [ITEMS, TILE, 3 * TILE])
def test_intersect_pairs_and_segments_around_borders(m):
    """A pair, and a segment start, at every row m - 8 .. m + 8; rows m - 1 and m sit in two threads (and tiles)."""
    for n in (m + 9, m + 20):
        for d in range(-8, 9):
            r = m + d
            if r < 1:
                continue
            start, stop = _no_pairs(n)
            stop[r - 1] = start[r] + 3                                   # row r pairs with the row before
            _sweep(start, stop, None, (n, r, "pair"))
            _sweep(start, stop, np.ones(n, np.uint8), (n, r, "pair, one segment"))
            same = np.ones(n, np.uint8)
            same[r] = 0
            _sweep(start, stop, same, (n, r, "pair cut by a segment start"))
            start, stop = _no_pairs(n)
            stop += 10                                                   # every row pairs
            _sweep(start, stop, same, (n, r, "every row, one segment start"))
            same[r - 1] = same[min(r + 1, n - 1)] = 0
            _sweep(start, stop, same, (n, r, "three segment starts"))


@pytest.mark.parametrize("n", [1, 2, ITEMS, TILE, TILE + 1, 5 * TILE + 3])
def test_intersect_every_row_none_and_no_segments(n):
    start, stop = _no_pairs(n)
    _sweep(start, stop, None, "none")
    _sweep(start, stop + 10, None, "every row")
    _sweep(start, stop + 10, np.zeros(n, np.uint8), "same_prev all zero")
    rng = np.random.default_rng(n)
    s = np.sort(rng.integers(0, 3 * n, n))
    e = np.sort(s + rng.integers(0, 8, n))
    _sweep(s, e, (rng.random(n) < 0.8).astype(np.uint8), "random")


def test_intersect_empty():
    _sweep(np.zeros(0, np.int64), np.zeros(0, np.int64), None, "empty")


@pytest.mark.parametrize("n", [20, 5 * TILE + 7])
def test_overlap_sums_past_2_32_and_2_63(n):
    """Positions near 2^59: every pair overlaps by about 2^59, so one block's sum passes 2^32 and the total passes
    2^63; the total wraps modulo 2^64 as NumPy's int64 sum does."""
    top = 1 << 59
    start = np.arange(n, dtype=np.int64)
    stop = top - n + np.arange(n, dtype=np.int64)
    _sweep(start, stop, None, "near 2^59")
    a = bnp.Interval(["chr1"] * n, start, stop)
    b = bnp.Interval(["chr1"] * n, start + 1, stop - 1)
    want = so.count_overlap(("x", start, stop), ("x", start + 1, stop - 1))
    assert count_overlap(a, b) == want
    mid = start * (1 << 20)
    assert count_overlap(bnp.Interval(["chr1"] * n, mid, mid + (1 << 40)), b) == \
        so.count_overlap(("x", mid, mid + (1 << 40)), ("x", start + 1, stop - 1))


# --------------------------------------------------------------------------------------------------------------------
# intersect against what it means
# --------------------------------------------------------------------------------------------------------------------
def _merged_set(rng, n, size, names):
    """A merged interval set (no two intervals of one chromosome overlap or touch), rows shuffled."""
    c, s, e = [], [], []
    for name in names:
        st = np.sort(rng.integers(0, size - 40, n))
        rows, stops = po.merge_intervals(st, st + rng.integers(1, 40, n))
        c += [name] * rows.size
        s.append(st[rows])
        e.append(stops)
    s, e = np.concatenate(s), np.concatenate(e)
    order = rng.permutation(s.size)
    return [c[i] for i in order], s[order], e[order]


def _iv(x):
    return bnp.Interval(list(x[0]), np.asarray(x[1], dtype=np.int64), np.asarray(x[2], dtype=np.int64))


def _rows(got):
    return list(zip(got.chromosome.tolist(), got.start.cpu().tolist(), got.stop.cpu().tolist()))


def _similarity(sizes, x, y, xy):
    n = sum(sizes.values())
    return float(Fraction(xy, x + y - xy)), float(Fraction(xy * n, x * y))


@pytest.mark.parametrize("n", [1, 50, 3000])
def test_intersect_is_the_intersection_of_merged_sets(n):
    rng = np.random.default_rng(60 + n)
    size = 12 * n + 100
    a, b = _merged_set(rng, n, size, ["chr1"]), _merged_set(rng, n, size, ["chr1"])
    ma, mb = po.dense_mask(a[1], a[2], size), po.dense_mask(b[1], b[2], size)
    got = intersect(_iv(a), _iv(b))
    ws, we = so.mask_intersect(a, b)["chr1"]
    assert sorted(_rows(got)) == [("chr1", int(x), int(y)) for x, y in zip(ws, we)]
    assert np.array_equal(get_boolean_mask(got, size).to_array().cpu().numpy(), ma & mb)
    assert count_overlap(_iv(a), _iv(b)) == int((ma & mb).sum())
    sizes = {"chr1": size}
    j, f = _similarity(sizes, int(ma.sum()), int(mb.sum()), int((ma & mb).sum()))
    assert jaccard(sizes, _iv(a), _iv(b)) == j
    if ma.any() and mb.any():
        assert forbes(sizes, _iv(a), _iv(b)) == f


@pytest.mark.parametrize("n", [5, 2000])
def test_global_intersect_is_the_intersection_on_every_chromosome(n):
    rng = np.random.default_rng(70 + n)
    names = ["chr1", "chr10", "chr2", "chrX", "chr1_alt"]
    sizes = {name: 12 * n + 100 for name in names}
    a, b = _merged_set(rng, n, 12 * n + 100, names), _merged_set(rng, n, 12 * n + 100, names[:4])
    got = global_intersect(_iv(b), _iv(a))
    want = so.mask_intersect(a, b)
    assert sorted(_rows(got)) == sorted((c, int(x), int(y)) for c, (s, e) in want.items() for x, y in zip(s, e))
    g = bnp.Genome.from_dict(sizes, filter_function=None)
    inter = g.get_intervals(got).get_mask()
    xa, xb, xab = 0, 0, 0
    for name in names:
        sel = [np.asarray(x[0]) == name for x in (a, b)]
        ma = po.dense_mask(a[1][sel[0]], a[2][sel[0]], sizes[name])
        mb = po.dense_mask(b[1][sel[1]], b[2][sel[1]], sizes[name])
        _check(inter[name], ma & mb, name)
        xa, xb, xab = xa + int(ma.sum()), xb + int(mb.sum()), xab + int((ma & mb).sum())
    j, f = _similarity(sizes, xa, xb, xab)
    assert jaccard(sizes, _iv(a), _iv(b)) == j and jaccard(g, _iv(a), _iv(b)) == j
    assert forbes(sizes, _iv(a), _iv(b)) == f


def test_global_intersect_ties_zero_length_and_long_last_stops():
    """Ties in start, zero-length rows, and a chromosome whose last stop lies past the next one's first start."""
    rng = np.random.default_rng(80)
    c, s, e = [], [], []
    for name, base in (("chr1", 0), ("chr2", 0), ("chr3", 500)):
        st = base + rng.integers(0, 300, 400)
        st[:40] = st[40:80]
        en = st + rng.integers(0, 30, 400)
        en[80:120] = st[80:120]
        en[-1] = 100_000                                   # past every start of the next chromosome
        c += [name] * 400
        s.append(st)
        e.append(en)
    s, e = np.concatenate(s), np.concatenate(e)
    half = len(c) // 2
    a, b = (c[:half], s[:half], e[:half]), (c[half:], s[half:], e[half:])
    for x, y in ((a, b), (b, a), (a, a)):
        got = global_intersect(_iv(y), _iv(x))
        rows, stops = so.global_intersect(y, x)
        names = list(x[0]) + list(y[0])
        starts = np.concatenate([x[1], y[1]])
        assert got.chromosome.tolist() == [names[r] for r in rows]
        assert got.start.cpu().tolist() == starts[rows].tolist() and got.stop.cpu().tolist() == stops.tolist()


# --------------------------------------------------------------------------------------------------------------------
# chromosome names past the first read's packing limits
# --------------------------------------------------------------------------------------------------------------------
def _named_rows(rng, distinct, n_runs):
    """Unsorted rows whose names change n_runs - 1 times (runs of 1 or 2 rows, cycling through ``distinct``)."""
    c = []
    for i in range(n_runs):
        c += [distinct[i % len(distinct)]] * int(rng.integers(1, 3))
    s = rng.integers(0, 1000, len(c))
    return c, s, s + rng.integers(0, 20, len(c))


def _runs_and_bytes(names):
    first = [i for i in range(len(names)) if i == 0 or names[i] != names[i - 1]]
    return len(first), sum(len(names[i].encode()) for i in first)


N256 = ["x" * 255 + ch for ch in "ab"]
NAME_CASES = {
    "runs_4095": (["chr1", "chr2", "chr10"], 4095),
    "runs_4096": (["chr1", "chr2", "chr10"], 4096),
    "runs_4097": (["chr1", "chr2", "chr10"], 4097),
    "runs_10000": (["chr1", "chr2", "chr10", "chrX"], 10_000),
    "bytes_mixed": (N256 + ["x" * 255], 256),         # 256 runs of 256 and 255 bytes: 65 451 bytes
    "bytes_65536": (N256, 256),                       # 256 runs of 256 bytes
    "bytes_65792": (N256, 257),
    "long_names": (["a", "b" * 10_000, "b" * 9_999], 10),
    "prefixes": (["c", "cc", "ccc", "c" * 40], 5000),
}


def _exact_bytes(rng, total):
    """Rows whose name runs total exactly ``total`` bytes: 256-byte names, then one shorter name."""
    c, n = [], 0
    while total - n >= 256:
        c.append(N256[len(c) % 2])
        n += 256
    if total > n:
        c.append("y" * (total - n))
    s = rng.integers(0, 1000, len(c))
    return c, s, s + 5


def _name_sets(case):
    rng = np.random.default_rng(len(case))
    if case.startswith("exact_"):
        return _exact_bytes(rng, int(case[6:]))
    return _named_rows(rng, *NAME_CASES[case])


@pytest.mark.parametrize("case", list(NAME_CASES) + ["exact_65535", "exact_65536", "exact_65537"])
def test_names_past_the_packing_limits(case):
    c, s, e = _name_sets(case)
    runs, nbytes = _runs_and_bytes(c)
    if case.startswith("runs_"):
        assert runs == int(case[5:])
    if case.startswith("exact_"):
        assert nbytes == int(case[6:])
    over = runs > NAME_SLOTS or nbytes > NAME_BYTES
    x = _iv((c, s, e))
    got, syncs = _count_syncs(lambda: sort_intervals(x))
    want = so.sort_intervals(c, s, e)
    assert got.chromosome.tolist() == [c[i] for i in want]
    assert got.start.cpu().tolist() == s[want].tolist() and got.stop.cpu().tolist() == e[want].tolist()
    assert syncs == 1 + over, (runs, nbytes, syncs)
    key = lambda n: len(n) // 3                                         # several names share a key
    got = sort_intervals(x, chromosome_key_function=key)
    want = so.sort_intervals(c, s, e, key=key)
    assert got.chromosome.tolist() == [c[i] for i in want] and got.start.cpu().tolist() == s[want].tolist()
    order = sorted(set(c), reverse=True)
    got = sort_intervals(x, sort_order=order)
    want = so.sort_intervals(c, s, e, sort_order=order)
    assert got.chromosome.tolist() == [c[i] for i in want] and got.stop.cpu().tolist() == e[want].tolist()
    with pytest.raises(KeyError):
        sort_intervals(x, sort_order=order[1:])
    # GenomicIntervals.sorted() in genome order
    sizes = {n: 2000 for n in order}
    g = bnp.Genome.from_dict(sizes, filter_function=None)
    got = g.get_intervals(x).sorted()
    want = so.sort_intervals(c, s, e, sort_order=list(sizes))
    assert got.chromosome.tolist() == [c[i] for i in want] and got.start.cpu().tolist() == s[want].tolist()
    # global_intersect of these rows with a small set, and jaccard
    rng = np.random.default_rng(runs)
    small = (order[:2] * 3, rng.integers(0, 1000, 6), None)
    small = (small[0], small[1], small[1] + 300)
    y = _iv(small)
    got, syncs = _count_syncs(lambda: global_intersect(y, x))
    rows, stops = so.global_intersect(small, (c, s, e))
    names = c + small[0]
    starts = np.concatenate([s, small[1]])
    assert got.chromosome.tolist() == [names[r] for r in rows]
    assert got.start.cpu().tolist() == starts[rows].tolist() and got.stop.cpu().tolist() == stops.tolist()
    assert syncs == 2 + over, (runs, nbytes, syncs)
    assert jaccard(sizes, x, _iv(small)) == so.jaccard(sizes, (c, s, e), small)
