"""Track operators, intersections, sorting and similarity of interval sets on the GPU against the NumPy oracle
(tests/interval_sets_oracle.py): every run, value, dtype and row must equal the oracle's."""
import gzip
import os
import warnings

import numpy as np
import pytest
import torch

import bionumpy_b200 as bnp
from bionumpy_b200 import _native as nv
from bionumpy_b200 import ops
from bionumpy_b200.arithmetics import (GenomicRunLengthArray, count_overlap, forbes, get_boolean_mask,
                                       get_contingency_table, global_intersect, intersect, jaccard, sort_intervals,
                                       unique_intersect)

import interval_sets_oracle as so
import pileup_oracle as po

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
TILE = 2048
I64 = np.iinfo(np.int64)

BINARY = [np.add, np.subtract, np.multiply, np.bitwise_and, np.bitwise_or, np.bitwise_xor, np.minimum, np.maximum,
          np.equal, np.not_equal, np.less, np.less_equal, np.greater, np.greater_equal, np.logical_and, np.logical_or,
          np.logical_xor]


def _track(dense):
    s, e, v = po.runs_of(dense)
    if dense.size == 0:
        return GenomicRunLengthArray(torch.zeros(2, dtype=torch.int64, device="cuda"),
                                     torch.zeros(1, dtype=torch.from_numpy(dense).dtype, device="cuda"), 0)
    return GenomicRunLengthArray.from_runs(s, e, torch.from_numpy(v))


def _check(got, want_dense):
    s, e, v = po.runs_of(want_dense)
    assert isinstance(got, GenomicRunLengthArray) and len(got) == want_dense.size
    assert got.dtype == torch.from_numpy(want_dense).dtype, (got.dtype, want_dense.dtype)
    if want_dense.size == 0:
        return
    assert got.starts.cpu().tolist() == s.tolist()
    assert got.ends.cpu().tolist() == e.tolist()
    assert got.values.cpu().tolist() == v.tolist()


def _random(rng, size, kind):
    if kind == "bool":
        return po.random_dense(rng, size, np.bool_)
    return po.random_dense(rng, size, np.int64)


def _expect(ufunc, *operands):
    try:
        return so.dense_op(ufunc, *operands)[0], None
    except TypeError as e:
        return None, e


@pytest.mark.parametrize("ufunc", BINARY, ids=lambda u: u.__name__)
@pytest.mark.parametrize("kinds", [("bool", "bool"), ("int", "int"), ("int", "bool"), ("int", "scalar"),
                                   ("scalar", "int"), ("bool", "scalar"), ("scalar", "bool")])
def test_every_operator(ufunc, kinds):
    rng = np.random.default_rng(BINARY.index(ufunc) * 100 + sum(map(ord, "".join(kinds))))
    size = 3000
    dense, args = [], []
    for k in kinds:
        if k == "scalar":
            v = [I64.max, -1, 0, True][rng.integers(4)]
            dense.append(v)
            args.append(v)
        else:
            d = _random(rng, size, k)
            dense.append(d)
            args.append(_track(d))
    want, err = _expect(ufunc, *dense)
    if err is not None:
        with pytest.raises(TypeError):
            ufunc(*args)
        return
    _check(ufunc(*args), want)


@pytest.mark.parametrize("kind", ["bool", "int"])
def test_unary_operators_and_python_operators(kind):
    rng = np.random.default_rng(5)
    d = _random(rng, 5000, kind)
    t = _track(d)
    _check(~t, ~d)
    _check(np.logical_not(t), np.logical_not(d))
    if kind == "int":
        _check(-t, -d)
    else:
        with pytest.raises(TypeError):
            -t
    e = _random(rng, 5000, kind)
    u = _track(e)
    for got, want in ((t & u, d & e), (t | u, d | e), (t ^ u, d ^ e), (t + u, d + e), (t * u, d * e),
                      (t == u, d == e), (t != u, d != e), (t < u, d < e), (t <= u, d <= e), (t > u, d > e),
                      (t >= u, d >= e), (t > 0, d > 0), (0 < t, 0 < d), (3 - t, 3 - so.widen(d)),
                      (np.maximum(t, u), np.maximum(d, e)), (np.minimum(1, t), np.minimum(1, d))):
        _check(got, so.widen(want) if want.dtype != np.bool_ else want)


def test_wrapping_extremes():
    d = np.repeat(np.array([I64.max, I64.min, -1, 0, 1, I64.max - 1], dtype=np.int64), 3)
    e = np.repeat(np.array([1, -1, I64.min, I64.max, I64.max, 2], dtype=np.int64), 3)
    t, u = _track(d), _track(e)
    for ufunc in (np.add, np.subtract, np.multiply):
        _check(ufunc(t, u), so.dense_op(ufunc, d, e)[0])
        _check(ufunc(t, I64.min), so.dense_op(ufunc, d, np.int64(I64.min))[0])
    _check(-t, so.dense_op(np.negative, d)[0])


@pytest.mark.parametrize("k", [1, 2, 5])
@pytest.mark.parametrize("delta", [-1, 0, 1])
def test_merged_counts_around_tile_borders(k, delta):
    """n_a + n_b = 2048 k - 1, 2048 k and 2048 k + 1 run starts."""
    rng = np.random.default_rng(k * 3 + delta)
    total = TILE * k + delta
    n_a = total // 3
    size = 10 * total
    a_starts = np.sort(rng.choice(np.arange(1, size), n_a - 1, replace=False))
    b_starts = np.sort(rng.choice(np.arange(1, size), total - n_a - 1, replace=False))
    d = np.repeat(np.arange(n_a) % 7, np.diff(np.concatenate([[0], a_starts, [size]])))
    e = np.repeat(np.arange(total - n_a) % 5, np.diff(np.concatenate([[0], b_starts, [size]])))
    ta = GenomicRunLengthArray.from_runs(np.concatenate([[0], a_starts]), np.concatenate([a_starts, [size]]),
                                         np.arange(n_a) % 7)
    tb = GenomicRunLengthArray.from_runs(np.concatenate([[0], b_starts]), np.concatenate([b_starts, [size]]),
                                         np.arange(total - n_a) % 5)
    assert ta.values.numel() + tb.values.numel() == total
    for ufunc in (np.add, np.equal, np.maximum):
        _check(ufunc(ta, tb), ufunc(d, e))


def test_all_of_a_before_b_and_identical_boundaries():
    size = 100_000
    a_starts = np.arange(0, 50_000, 7)
    d = np.repeat(np.arange(a_starts.size) % 3, np.diff(np.concatenate([a_starts, [size]])))
    b_starts = np.concatenate([[0], np.arange(50_000, size, 11)])
    e = np.repeat(np.arange(b_starts.size) % 4, np.diff(np.concatenate([b_starts, [size]])))
    _check(_track(d) + _track(e), d + e)
    _check(_track(d) - _track(d), d - d)                     # identical boundaries: one run of 0
    _check(_track(d) * _track(d + 1), d * (d + 1))


def test_one_run_against_a_million_runs():
    rng = np.random.default_rng(7)
    size = 3_000_000
    d = po.random_dense(rng, size, np.int64, max_run=3)
    t = _track(d)
    assert t.values.numel() > 1_000_000
    _check(t + 5, d + 5)
    _check(np.maximum(7, t), np.maximum(7, d))
    _check(t >= -1000, d >= -1000)


def test_constant_result_spanning_many_tiles():
    rng = np.random.default_rng(8)
    size = 2_000_000
    d = po.random_dense(rng, size, np.int64, max_run=2)
    t = _track(d)
    assert t.values.numel() > 300 * TILE
    for got in (t - t, t == t, t ^ t, np.logical_or(t, True)):
        assert got.values.numel() == 1 and got.starts.cpu().tolist() == [0] and got.ends.cpu().tolist() == [size]


def test_non_canonical_inputs_from_astype():
    rng = np.random.default_rng(9)
    d = po.random_dense(rng, 20_000, np.int64)
    t = _track(d).astype(bool)                              # neighbouring runs with equal values
    assert t.values.numel() > len(po.runs_of(d != 0)[0])
    e = po.random_dense(rng, 20_000, np.bool_)
    _check(t & _track(e), (d != 0) & e)
    _check(t | False, d != 0)
    n = _track(np.clip(d, -100, 100).astype(np.int8))
    _check(n.astype(np.int16) + 1, np.clip(d, -100, 100).astype(np.int64) + 1)
    _check(np.logical_and(_track(d), 3), np.logical_and(d, 3))


def test_size_zero_and_size_mismatch():
    z = _track(np.zeros(0, dtype=np.int64))
    out = z + z
    assert len(out) == 0 and out.dtype == torch.int64
    assert len(z == 0) == 0 and (z == 0).dtype == torch.bool
    with pytest.raises(ValueError):
        _track(np.zeros(3, dtype=np.int64)) + _track(np.zeros(4, dtype=np.int64))


def test_dense_fallback_keeps_numpy_results():
    d = np.array([1, 1, 4, 4, 9], dtype=np.int64)
    t = _track(d)
    assert np.sqrt(t).tolist() == np.sqrt(d).tolist()
    assert (t + 0.5).tolist() == (d + 0.5).tolist()
    assert np.add.reduce(t) == d.sum()


# --------------------------------------------------------------------------------------------------------------------
# genome tracks
# --------------------------------------------------------------------------------------------------------------------
def _bed(name):
    return po.parse_bed(gzip.open(os.path.join(GOLDEN, name)).read())


@pytest.fixture(scope="module")
def hg38():
    return bnp.Genome.from_file(os.path.join(GOLDEN, "hg38.chrom.sizes"))


def test_genomic_array_masks_on_hg38(hg38):
    ctcf = hg38.read_intervals(os.path.join(GOLDEN, "ctcf.bed.gz"))
    znf = hg38.read_intervals(os.path.join(GOLDEN, "znf263.bed.gz"))
    ma, mb = ctcf.get_mask(), znf.get_mask()
    both, either = ma & mb, ma | mb
    sizes = po.read_sizes(open(os.path.join(GOLDEN, "hg38.chrom.sizes")).read())
    keep = {n: v for n, v in sizes.items() if "_" not in n}
    a = [np.asarray(x) for x in _bed("ctcf.bed.gz")]
    b = [np.asarray(x) for x in _bed("znf263.bed.gz")]
    a = (list(a[0][np.isin(a[0], list(keep))]), a[1][np.isin(a[0], list(keep))], a[2][np.isin(a[0], list(keep))])
    b = (list(b[0][np.isin(b[0], list(keep))]), b[1][np.isin(b[0], list(keep))], b[2][np.isin(b[0], list(keep))])
    ((x, y), (z, w)) = so.contingency_table(a, b, hg38.size)
    assert int(both.sum()) == x and int(either.sum()) == x + y + z
    assert both.dtype == torch.bool
    # the canonical runs of the intersection equal the combined dense masks of one contig
    da, db = ma["chr21"].to_array().cpu().numpy(), mb["chr21"].to_array().cpu().numpy()
    _check(both["chr21"], da & db)
    other = bnp.Genome.from_dict({"chr1": 10})
    with pytest.raises(ValueError):
        ma & other.get_intervals(bnp.Interval(["chr1"], [1], [3])).get_mask()
    with pytest.raises(TypeError):
        ma - mb


# --------------------------------------------------------------------------------------------------------------------
# intersect, global_intersect and count_overlap
# --------------------------------------------------------------------------------------------------------------------
def _iv(chroms, starts, stops):
    return bnp.Interval(list(chroms), np.asarray(starts, dtype=np.int64), np.asarray(stops, dtype=np.int64))


def _check_rows(got, a, b, rows, stops):
    names = list(a[0]) + list(b[0])
    starts = np.concatenate([a[1], b[1]])
    assert got.chromosome.tolist() == [names[r] for r in rows]
    assert got.start.cpu().tolist() == starts[rows].tolist()
    assert got.stop.cpu().tolist() == stops.tolist()


def _random_sets(rng, n, size, names=("chr1",)):
    out = []
    for m in (n, n // 2 + 1):
        c = [names[i] for i in rng.integers(0, len(names), m)]
        s = rng.integers(0, size, m)
        e = s + rng.integers(0, 40, m)
        s[: m // 10] = s[m // 10: 2 * (m // 10)]                    # ties in start
        e[m // 10: m // 5] = s[m // 10: m // 5]                     # zero-length
        out.append((c, s, e))
    return out


@pytest.mark.parametrize("n", [1, 3, 1000, TILE - 1, TILE, 3 * TILE + 5])
def test_intersect_against_oracle(n):
    rng = np.random.default_rng(n)
    a, b = _random_sets(rng, n, 5 * n + 10)
    got = intersect(_iv(*a), _iv(*b))
    _check_rows(got, a, b, *so.intersect(a, b))
    assert count_overlap(_iv(*a), _iv(*b)) == so.count_overlap(a, b)


def test_intersect_ties_touching_and_zero_length():
    a = (["chr1"] * 4, np.array([10, 10, 20, 30]), np.array([15, 12, 25, 30]))
    b = (["chr1"] * 3, np.array([10, 25, 29]), np.array([11, 26, 31]))
    got = intersect(_iv(*a), _iv(*b))
    rows, stops = so.intersect(a, b)
    _check_rows(got, a, b, rows, stops)
    assert 5 not in rows.tolist()                         # 25-26 only touches 20-25: not emitted
    assert rows.tolist()[:2] == [1, 4]                    # the stable order of the three rows at 10
    assert count_overlap(_iv(*a), _iv(*b)) == so.count_overlap(a, b)


def test_intersect_reference_golden():
    a = _iv(["chr1"] * 3, [10, 20, 30], [15, 29, 35])
    b = _iv(["chr1"] * 3, [10, 22, 29], [15, 28, 36])
    got = intersect(a, b)
    assert got.start.cpu().tolist() == [10, 22, 30] and got.stop.cpu().tolist() == [15, 28, 35]
    assert count_overlap(a, b) == 16
    with pytest.raises(TypeError):
        intersect(a, bnp.Bed6(["chr1"], [1], [2], ["x"], [0], ["+"]))


def test_one_million_rows():
    rng = np.random.default_rng(11)
    a, b = _random_sets(rng, 1_000_000, 50_000_000)
    got = intersect(_iv(*a), _iv(*b))
    _check_rows(got, a, b, *so.intersect(a, b))
    assert count_overlap(_iv(*a), _iv(*b)) == so.count_overlap(a, b)


@pytest.mark.parametrize("n", [5, 2000, 3 * TILE + 1])
def test_global_intersect_multi_chromosome(n):
    rng = np.random.default_rng(n + 1)
    a, b = _random_sets(rng, n, 3 * n, names=("chr1", "chr10", "chr2", "chrX"))
    got = global_intersect(_iv(*b), _iv(*a))
    _check_rows(got, a, b, *so.global_intersect(b, a))


def test_global_intersect_does_not_cross_chromosomes():
    a = (["chr1"], np.array([100]), np.array([200]))
    b = (["chr2"], np.array([10]), np.array([20]))
    assert len(global_intersect(_iv(*b), _iv(*a))) == 0
    assert len(global_intersect(_iv(*a), _iv(*b))) == 0


# --------------------------------------------------------------------------------------------------------------------
# sorting, unique_intersect, similarity
# --------------------------------------------------------------------------------------------------------------------
def test_sort_intervals():
    d = (["chr3", "chr2", "chr2", "chr1"], np.array([10, 15, 14, 12]), np.array([20, 22, 23, 24]))
    assert sort_intervals(_iv(*d)).start.cpu().tolist() == [12, 14, 15, 10]
    rng = np.random.default_rng(12)
    names = ["chr%d" % i for i in (1, 2, 10, 11, 3)] + ["chrX"]
    c = [names[i] for i in rng.integers(0, len(names), 5000)]
    s = rng.integers(0, 100, 5000)
    e = s + rng.integers(0, 5, 5000)
    key = lambda n: (not n[3:].isdigit(), int(n[3:]) if n[3:].isdigit() else n)
    order = names[::-1]
    for kwargs in ({}, {"chromosome_key_function": key}, {"sort_order": order}):
        got = sort_intervals(_iv(c, s, e), **kwargs)
        want = so.sort_intervals(c, s, e, **{k.replace("chromosome_key_function", "key"): v for k, v in kwargs.items()})
        assert got.chromosome.tolist() == [c[i] for i in want]
        assert got.start.cpu().tolist() == s[want].tolist() and got.stop.cpu().tolist() == e[want].tolist()
    with pytest.raises(KeyError):
        sort_intervals(_iv(c, s, e), sort_order=names[:-1])


def test_genomic_intervals_sorted():
    g = bnp.Genome.from_dict({"chr2": 100, "chr1": 100, "chr10": 100})
    c = ["chr1", "chr10", "chr2", "chr1", "chr2", "chr1"]
    s = np.array([5, 1, 7, 5, 0, 2])
    e = np.array([9, 3, 8, 6, 100, 2])
    got = g.get_intervals(_iv(c, s, e)).sorted()
    want = so.sort_intervals(c, s, e, sort_order=["chr2", "chr1", "chr10"])
    assert got.chromosome.tolist() == [c[i] for i in want] and got.start.cpu().tolist() == s[want].tolist()
    assert got.stop.cpu().tolist() == e[want].tolist()


def test_unique_intersect():
    small = _iv(["chr1"] * 4, [2, 5, 10, 11], [5, 7, 12, 13])
    got = unique_intersect(small, _iv(["chr1"], [7], [11]), 20)
    assert got.start.cpu().tolist() == [10] and got.stop.cpu().tolist() == [12]


def test_unique_intersect_example_chain():
    """scripts/unique_intersect_example.py: 3951 ctcf peaks meet a znf263 peak on hg38."""
    genome = bnp.Genome.from_file(os.path.join(GOLDEN, "hg38.chrom.sizes"), filter_function=None)
    mask = genome.read_intervals(os.path.join(GOLDEN, "znf263.bed.gz")).get_mask()
    ctcf = bnp.open(os.path.join(GOLDEN, "ctcf.bed.gz")).read()
    kept = ctcf[mask[ctcf].any(axis=-1)]
    want = so.unique_intersect(_bed("ctcf.bed.gz"), _bed("znf263.bed.gz"))
    assert len(kept) == 3951 and kept.start.cpu().tolist() == _bed("ctcf.bed.gz")[1][want].tolist()


def test_similarity_goldens():
    a = _iv(["chr1", "chr2"], [10, 20], [20, 30])
    b = _iv(["chr1", "chr2"], [15, 15], [22, 25])
    sizes = {"chr1": 100, "chr2": 50}
    assert forbes(sizes, a, b) == (150 * 10) / (20 * 17)
    assert jaccard(sizes, a, b) == 10 / (12 + 15)
    assert get_contingency_table(_iv(["chr1"], [10], [20]), _iv(["chr1"], [15], [22]), 100) == [[5, 5], [2, 88]]
    a = _iv(["chr1", "chr2"], [10, 20], [20, 30])
    b = _iv(["chr2", "chr1"], [15, 10], [25, 40])
    assert forbes({"chr1": 100, "chr2": 200}, a, b) == 5.625
    with pytest.raises(KeyError):
        jaccard({"chr1": 100}, a, b)


def test_jaccard_and_forbes_on_hg38():
    sizes = po.read_sizes(open(os.path.join(GOLDEN, "hg38.chrom.sizes")).read())
    genome = bnp.Genome.from_dict(sizes, filter_function=None)
    a, b = _bed("ctcf.bed.gz"), _bed("znf263.bed.gz")
    ia = bnp.open(os.path.join(GOLDEN, "ctcf.bed.gz")).read()
    ib = bnp.open(os.path.join(GOLDEN, "znf263.bed.gz")).read()
    assert jaccard(genome, ia, ib) == so.jaccard(sizes, a, b)
    assert forbes(sizes, ia, ib) == so.forbes(sizes, a, b)


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


def test_synchronisations_and_launch_counts():
    lib = nv.load_library()
    launches = []
    sizes = {"chr1": 60_000_000, "chr2": 1000}
    genome = bnp.Genome.from_dict(sizes)
    for n in (10, 200_000):
        rng = np.random.default_rng(n)
        a, b = _random_sets(rng, n, 900, names=("chr1", "chr2"))
        a, b = ((sorted(x[0]), x[1], x[1] + rng.integers(0, 50, x[1].size)) for x in (a, b))   # names in runs, as in BED
        ia, ib = _iv(*a), _iv(*b)
        ma, mb = get_boolean_mask(ia, 1000), get_boolean_mask(ib, 1000)
        pa = get_boolean_mask(ia, 1000).astype(int)
        for fn, want in ((lambda: ma & mb, 1), (lambda: pa > 0, 1), (lambda: ~ma, 1), (lambda: intersect(ia, ib), 1),
                         (lambda: count_overlap(ia, ib), 1), (lambda: sort_intervals(ia), 1),
                         (lambda: global_intersect(ib, ia), 2), (lambda: unique_intersect(ia, ib, 1000), 2)):
            before = lib.bnpk_launch_count()
            _, syncs = _count_syncs(fn)
            launches.append((n, lib.bnpk_launch_count() - before))
            assert syncs == want, (fn, syncs)
        genome._name_table()
        _, syncs = _count_syncs(lambda: jaccard(genome, ia, ib))
        assert syncs <= 6
    assert [c for n, c in launches if n == 10] == [c for n, c in launches if n == 200_000], launches


def test_dispatcher_ops():
    torch.ops.load_library(os.path.join(os.path.dirname(nv.LIB_PATH), "libbnpk_torch.so"))
    a = torch.tensor([0, 3, 10], device="cuda")
    av = torch.tensor([1, 2], device="cuda")
    b = torch.tensor([0, 5, 10], device="cuda")
    bv = torch.tensor([2, 2], device="cuda")
    s, v, n = torch.ops.bnpk.runs_combine(a, av, b, bv, nv.OP_EQ)
    k = int(n[0])
    assert (s[:k + 1].tolist(), v[:k].tolist()) == ([0, 3, 10], [0, 1])
    s2, v2, n2 = ops.runs_combine(a, av, b, bv, nv.OP_EQ)
    assert int(n2[0]) == k and s2[:k + 1].tolist() == s[:k + 1].tolist()
    st = torch.tensor([1, 2, 8], device="cuda")
    sp = torch.tensor([5, 6, 9], device="cuda")
    rows, stops, n_out, over = torch.ops.bnpk.interval_intersect(st, sp, None, True)
    assert int(n_out[0]) == 1 and rows[:1].tolist() == [1] and stops[:1].tolist() == [5] and int(over[0]) == 3
    _, _, n_out, over = torch.ops.bnpk.interval_intersect(st, sp, None, False)
    assert int(n_out[0]) == 1 and int(over[0]) == 3
