"""bedGraph and float64 tracks on the GPU against tests/bedgraph_oracle.py and dense NumPy: the device decimal parser
bit for bit against float() (a million random texts, every digit count, the whole exponent range, hard cases, every
rejected form), bedGraph reading (chunk views at every offset with poison after them, CRLF, track/browser headers, whole
and chunked reads, gzip and BGZF), get_track (order, gaps, merging, -0.0, every error, one synchronisation), the fused
float reductions, every float operator and operand kind, and the guide's and the treat/control workflows."""
import gzip
import math
import os
import random
import warnings

import numpy as np
import pytest
import torch

import bam_oracle as bo
import bedgraph_oracle as oracle
import bionumpy_b200 as bnp
from bionumpy_b200 import _native as nv
from bionumpy_b200 import ops, torch_ops
from bionumpy_b200.arithmetics import FloatRunLengthArray, GenomicRunLengthArray
from bionumpy_b200.genomic_data.genome import GenomicArray, ignore_underscores
from bionumpy_b200.io.decimal import pow5_table
from bionumpy_b200.io.delimited import BdgBuffer, BedGraphBuffer
from bionumpy_b200.io.exceptions import FormatException

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
GUIDE_MAX = [227, 231, 412, 296, 165, 163, 271, 148, 268, 568, 1901, 90, 236]
GUIDE_MEAN = [145.68181818, 147.86129032, 256.671875, 187.71202532, 106.79934211, 106.23355263, 173.04501608,
              96.27152318, 169.59235669, 346.37272727, 593.44084507, 60.25614035, 150.72580645]


def _golden(name):
    return os.path.join(GOLDEN, name)


def bits(values):
    """int64 bit patterns, every NaN as one pattern (NaN equals NaN)."""
    a = np.asarray(values, dtype=np.float64).copy()
    a[np.isnan(a)] = np.nan
    return a.view(np.int64)


def _device_text(texts):
    data = b"".join(texts)
    base = torch.from_numpy(np.frombuffer(data + b"\0", dtype=np.uint8).copy()).cuda()
    lens = np.array([len(t) for t in texts], dtype=np.int64)
    starts = np.concatenate([[0], np.cumsum(lens)[:-1]]).astype(np.int64)
    return base, torch.from_numpy(starts).cuda(), torch.from_numpy(lens.astype(np.int32)).cuda()


def parse_all(texts):
    base, starts, lens = _device_text([t.encode() for t in texts])
    values, status = ops.parse_float(base, starts, lens, 3, pow5_table(base.device))
    return values.cpu().numpy(), ops.read_status(status)


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


# --------------------------------------------------------------------------------------------------------------------
# the parser
# --------------------------------------------------------------------------------------------------------------------
HARD = ["9007199254740993", "2.2250738585072011e-308", "4.9406564584124654e-324", "1.7976931348623157e308",
        "1.7976931348623159e308", "2.4703282292062327e-324", "2.4703282292062328e-324", "-0", "-0.0e5", "+.5", "5.",
        "0.1", "1e23", "8.98846567431158e307", "9007199254740992.5", "9007199254740993.0", "4503599627370496.5",
        "1e-400", "-1e400", "1e0000000000000000000000000001", "0." + "0" * 400 + "1", "1" + "0" * 400,
        "1234567890123456789", "0.000000001234567890123456789e300", "2.225073858507201e-308",
        "7.2057594037927933e16", "1.00000000000000011102230246251565404236316680908203125e0"[:21],
        "123456789012345678900000000", "1.5000000000000000000000000"]


def random_texts(rng, n):
    out = []
    for _ in range(n):
        nd = rng.randint(1, 19)
        digits = str(rng.randint(10 ** (nd - 1), 10 ** nd - 1))
        point = rng.randint(0, nd)
        form = rng.random()
        if form < 0.3:
            text = digits[:point] + "." + digits[point:] if point < nd else digits
        elif form < 0.5:
            text = "0" * rng.randint(0, 3) + digits + ("." if rng.random() < 0.2 else "")
        else:
            mant = digits[:point] + "." + digits[point:] if point < nd else digits
            if mant.startswith("."):
                mant = mant if rng.random() < 0.5 else "0" + mant
            e = rng.randint(-345, 310)
            text = mant + rng.choice("eE") + rng.choice(["", "+", "-"] if e >= 0 else ["-"]) + str(abs(e))
        out.append(rng.choice(["", "", "-", "+"]) + text)
    return out


def test_parse_matches_float_bit_for_bit():
    rng = random.Random(7)
    texts = HARD + random_texts(rng, 1_000_000)
    for nd in range(1, 20):                                  # every digit count, at both ends of the double range
        for e in (-340, -320, -308, -300, -22, -1, 0, 15, 22, 23, 290, 308):
            texts.append(str(rng.randint(10 ** (nd - 1), 10 ** nd - 1)) + "e" + str(e - nd))
    got, st = parse_all(texts)
    assert st.fault is None
    want = np.array([float(t) for t in texts])
    for t in texts[:len(HARD)]:
        assert oracle.parse(t) == float(t)
    bad = np.nonzero(got.view(np.int64) != want.view(np.int64))[0]
    assert bad.size == 0, [(texts[i], got[i], want[i]) for i in bad[:10]]
    assert got[texts.index("1.7976931348623159e308")] == math.inf
    assert np.signbit(got[texts.index("-0")])


REJECTED = ["", ".", "+", "-", "e5", "1e", "1e+", "1.2.3", "nan", "NaN", "inf", "-inf", "Infinity", "0x1p3", "1_000",
            " 1", "1 ", "+-1", "1e5.0", "12345678901234567891", "1.2345678901234567891", "--1", "1,5"]


def test_every_rejected_form_is_a_fault_of_its_row():
    for text in REJECTED:
        with pytest.raises(ValueError):
            oracle.parse(text)
        _, st = parse_all(["1.5", "2", text, "3"])
        assert st.column_fault() == (2, 3, nv.BAD_FLOAT), text
        data = ("c\t0\t1\t1.5\nc\t1\t2\t" + text + "\nc\t2\t3\t4\n").encode()
        with pytest.raises(FormatException) as err:
            BedGraphBuffer.from_raw_buffer(bnp.as_encoded_array(data.decode("utf-8")))
        assert err.value.line_number == 1 and "significant digits" in str(err.value), text
    # at most 19 significant digits: leading zeros and trailing zeros of the significand are not counted
    for text in ["0000001234567890123456789", "1234567890123456789000000", "0.1234567890123456789000"]:
        got, st = parse_all([text])
        assert st.fault is None and got[0] == float(text)


# --------------------------------------------------------------------------------------------------------------------
# reading bedGraph
# --------------------------------------------------------------------------------------------------------------------
def _text_rows(bg):
    data = bg.chromosome.ravel().raw().cpu().numpy().tobytes()
    ends = np.cumsum(bg.chromosome.lengths.cpu().numpy().astype(np.int64))
    names = [data[a:b].decode() for a, b in zip(np.concatenate([[0], ends[:-1]]), ends)]
    values = bg.value.cpu().numpy()
    assert bg.value.dtype == torch.float64
    return list(zip(names, bg.start.cpu().tolist(), bg.stop.cpu().tolist(), bits(values).tolist()))


def _oracle_rows(path):
    return [(c, s, e, int(bits([v])[0])) for c, s, e, v in oracle.read_bedgraph(path)]


@pytest.mark.parametrize("name", ["small_treat_pileup.bdg", "small.bdg"])
def test_fixture_whole_chunked_and_gzipped(name, tmp_path):
    path = _golden(name)
    want = _oracle_rows(path)
    assert _text_rows(bnp.open(path).read()) == want
    for size in (97, 4096):
        with bnp.open(path) as f:
            assert sum((_text_rows(c) for c in f.read_chunks(min_chunk_size=size)), []) == want
    data = open(path, "rb").read()
    for fname, raw in (("x.bdg.gz", gzip.compress(data)), ("y.bdg.gz", bo.bgzf(data, block=1000))):
        p = str(tmp_path / fname)
        open(p, "wb").write(raw)
        assert _text_rows(bnp.open(p).read()) == want
        with bnp.open(p) as f:
            assert sum((_text_rows(c) for c in f.read_chunks(min_chunk_size=500)), []) == want


def test_headers_crlf_and_every_line_border(tmp_path):
    body = open(_golden("small.bdg"), "rb").read().split(b"\n", 1)[1]
    want = [(c, s, e, int(bits([v])[0])) for c, s, e, v in oracle.read_bedgraph(_golden("small.bdg"))]
    head = b"track type=bedGraph name=x\nbrowser position chr1:1-100\n#c\n"
    for raw in (head + body, (head + body).replace(b"\n", b"\r\n")):
        p = str(tmp_path / "h.bdg")
        open(p, "wb").write(raw)
        assert _text_rows(bnp.open(p).read()) == want
    lines = body.split(b"\n")[:-1]
    for k in range(0, len(lines), 7):
        cut = b"".join(x + b"\n" for x in lines[:k]) + lines[k][:3]
        if k == 0:
            continue
        buf = BedGraphBuffer.from_raw_buffer(bnp.as_encoded_array(cut.decode()))
        assert buf.size == len(b"".join(x + b"\n" for x in lines[:k]))
        assert _text_rows(buf.get_data()) == want[:k]


def test_chunk_views_at_every_offset_with_poison_after():
    body = open(_golden("small.bdg"), "rb").read().split(b"\n", 1)[1]
    want = [(c, s, e, int(bits([v])[0])) for c, s, e, v in oracle.read_bedgraph(_golden("small.bdg"))]
    poison = b"1234567.89e12" * 8
    for off in range(16):
        raw = b"9" * off + body + poison
        big = torch.from_numpy(np.frombuffer(raw, dtype=np.uint8).copy()).cuda()
        buf = BedGraphBuffer.from_raw_buffer(big[off:off + len(body)])
        assert buf.size == len(body)
        assert _text_rows(buf.get_data()) == want


def test_bad_lines_name_their_line():
    for data, line in (("a\t0\t1\t1\nb\t1\t2\n", 1), ("a\t0\t1\tx\n", 0), ("a\t0\t1\t1\na\t1\t2\t2\na\t2\t3\t1e\n", 2)):
        with pytest.raises(FormatException) as err:
            BedGraphBuffer.from_raw_buffer(bnp.as_encoded_array(data))
        assert err.value.line_number == line


# --------------------------------------------------------------------------------------------------------------------
# get_track
# --------------------------------------------------------------------------------------------------------------------
def _dense(track, genome):
    return {name: np.asarray(track[name]) for name in genome.get_chromosome_sizes()}


def _canonical(t):
    v = bits(t.values.cpu().numpy()) if t.values.is_floating_point() else t.values.cpu().numpy()
    s = t.starts.cpu().numpy()
    assert s[0] == 0 and np.all(np.diff(np.append(s, t.ends.cpu().numpy()[-1:])) > 0)
    if t.values.is_floating_point():
        raw = t.values.cpu().numpy().view(np.int64)
        assert np.all(raw[1:] != raw[:-1])
    else:
        assert np.all(v[1:] != v[:-1])


def test_get_track_rows_in_any_order_gaps_merges_and_signed_zero():
    genome = bnp.Genome.from_dict({"a": 100, "b": 50, "c_alt": 30}, filter_function=ignore_underscores)
    rows = [("a", 0, 10, 1.5), ("a", 10, 20, 1.5), ("a", 30, 40, -0.0), ("a", 40, 45, 0.0), ("b", 5, 5, 7.0),
            ("b", 10, 50, 2.0), ("a", 90, 100, math.inf), ("c_alt", 0, 10, 3.0), ("a", 20, 25, math.nan)]
    order = [8, 3, 0, 6, 2, 5, 1, 4, 7]
    shuffled = [rows[i] for i in order]
    bg = bnp.BedGraph([r[0] for r in shuffled], [r[1] for r in shuffled], [r[2] for r in shuffled],
                      np.array([r[3] for r in shuffled]))
    track = genome.get_track(bg)
    assert isinstance(track._global, FloatRunLengthArray)
    want = oracle.dense_track([r for r in rows if r[0] != "c_alt"], {"a": 100, "b": 50})
    dense = _dense(track, genome)
    for name in ("a", "b"):
        assert np.array_equal(bits(dense[name]), bits(want[name])), name
    _canonical(track._global)
    # [0, 20) is one run; -0.0 and +0.0 are two runs; the gap after it is +0.0 and merges with [40, 45)
    a = track["a"]
    assert a.starts.cpu().tolist()[:6] == [0, 20, 25, 30, 40, 90]


def test_get_track_errors_empty_and_integer_input():
    genome = bnp.Genome.from_dict({"a": 100, "b": 50})
    def bg(rows):
        return bnp.BedGraph([r[0] for r in rows], [r[1] for r in rows], [r[2] for r in rows],
                            np.array([float(r[3]) for r in rows]))
    with pytest.raises(ValueError, match="overlap"):
        genome.get_track(bg([("a", 50, 60, 1), ("a", 0, 10, 1), ("a", 55, 70, 2)]))
    with pytest.raises(ValueError, match="row 1"):
        genome.get_track(bg([("a", 0, 10, 1), ("a", 20, 10, 1)]))
    with pytest.raises(ValueError, match="row 0"):
        genome.get_track(bg([("b", 40, 60, 1)]))
    with pytest.raises(KeyError):
        genome.get_track(bg([("a", 0, 10, 1), ("zz", 0, 10, 1)]))
    empty = genome.get_track(bnp.BedGraph([], [], [], np.zeros(0)))
    assert np.array_equal(np.asarray(empty["a"]), np.zeros(100)) and empty.dtype == torch.float64
    ints = bnp.BedGraph(["a", "a", "b"], [0, 10, 0], [5, 15, 5], [1, 2, 3])
    t = bnp.Genome.from_dict({"a": 20, "b": 10}).get_track(ints)
    assert t.dtype == torch.int64
    assert str(t) == "a: [1 1 1 1 1 0 0 0 0 0 2 2 2 2 2 0 0 0 0 0]\nb: [3 3 3 3 3 0 0 0 0 0]"


def test_get_track_synchronises_once():
    genome = bnp.Genome.from_dict({"a": 10_000_000, "b": 1000})
    rng = np.random.default_rng(3)
    cuts = np.sort(rng.choice(10_000_000, 20_000, replace=False))
    bg = bnp.BedGraph(["a"] * 10_000, cuts[0::2], cuts[1::2], rng.random(10_000))
    torch.cuda.synchronize()
    lib = nv.load_library()
    n0 = lib.bnpk_launch_count()
    track, syncs = _count_syncs(lambda: genome.get_track(bg))
    assert syncs == 1
    # the name lookup and the bounds check, each with its status block's initialisation
    assert lib.bnpk_launch_count() - n0 == 4
    want = oracle.dense_track(list(zip(["a"] * 10_000, cuts[0::2].tolist(), cuts[1::2].tolist(),
                                       bg.value.cpu().tolist())), {"a": 10_000_000, "b": 1000})
    assert np.array_equal(bits(np.asarray(track["a"])), bits(want["a"]))


# --------------------------------------------------------------------------------------------------------------------
# reductions
# --------------------------------------------------------------------------------------------------------------------
SPECIAL = [math.nan, math.inf, -math.inf, 0.0, -0.0]


def random_track(rng, size, n_runs, special=0.05):
    cuts = np.sort(rng.choice(np.arange(1, size), n_runs - 1, replace=False))
    starts = np.concatenate([[0], cuts]).astype(np.int64)
    values = rng.normal(0, 100, n_runs)
    mask = rng.random(n_runs) < special
    values[mask] = rng.choice(SPECIAL, mask.sum())
    # canonical: no two neighbours with the same bits
    keep = np.concatenate([[True], bits(values)[1:] != bits(values)[:-1]]) | np.isnan(values)
    keep[1:] &= ~(np.isnan(values[1:]) & np.isnan(values[:-1]))
    starts, values = starts[keep], values[keep]
    return FloatRunLengthArray.from_runs(starts, np.append(starts[1:], size), values)


def _check_reductions(track, dense, q0, q1):
    rows = track[bnp.Interval(["x"] * len(q0), q0, q1)]
    got = {m: getattr(rows, m)(axis=-1).cpu().numpy() for m in ("max", "min", "sum", "mean", "any")}
    again = {m: getattr(rows, m)(axis=-1).cpu().numpy() for m in ("sum", "mean", "max")}
    starts = track.starts.cpu().numpy()
    for i, (a, b) in enumerate(zip(q0, q1)):
        a, b = max(a, 0), min(b, len(dense))
        seg = dense[a:b] if b > a else dense[:0]
        if seg.size == 0:
            assert got["max"][i] == -math.inf and got["min"][i] == math.inf and got["sum"][i] == 0
            assert math.isnan(got["mean"][i]) and not got["any"][i]
            continue
        assert bits([got["max"][i]]) == bits([np.max(seg)]) or got["max"][i] == np.max(seg)
        assert bits([got["min"][i]]) == bits([np.min(seg)]) or got["min"][i] == np.min(seg)
        assert bool(got["any"][i]) == bool(np.any(seg))
        if np.isnan(seg).any() or (np.isinf(seg).any() and (seg == math.inf).any() and (seg == -math.inf).any()):
            assert math.isnan(got["sum"][i]) and math.isnan(got["mean"][i])
            continue
        if np.isinf(seg).any():
            assert got["sum"][i] == np.sum(seg)
            continue
        n_runs = np.searchsorted(starts, b, "left") - np.searchsorted(starts, a, "right") + 1
        exact = oracle.exact_sum(seg)
        bound = 2 * n_runs * 2.0 ** -53 * float(sum(abs(x) for x in seg)) + 1e-300
        assert abs(float(exact) - got["sum"][i]) <= bound, (i, float(exact), got["sum"][i])
        assert abs(float(exact) / (b - a) - got["mean"][i]) <= bound / (b - a) + abs(float(exact) / (b - a)) * 2 ** -52
    for m in again:
        assert np.array_equal(bits(got[m]), bits(again[m])), m


def test_reductions_against_the_oracle():
    rng = np.random.default_rng(11)
    size = 300_000
    track = random_track(rng, size, 20_000)
    dense = np.asarray(track)
    q0 = rng.integers(-50, size, 2000)
    q1 = q0 + rng.integers(0, 400, 2000)
    q0 = np.concatenate([q0, [0, 5, 0, size - 10, size + 5, -100, 1000]])
    q1 = np.concatenate([q1, [size, 5, size + 100, size + 10, size + 10, 10, 999]])
    _check_reductions(track, dense, q0.tolist(), q1.tolist())


def test_long_queries_have_the_same_bits_every_time():
    rng = np.random.default_rng(5)
    size = 5_000_000
    track = random_track(rng, size, 800_000, special=0.0)
    dense = np.asarray(track)
    q0, q1 = [0, 1, 17, 2_000_000], [size, size - 1, 4_000_000, 2_000_003]
    _check_reductions(track, dense, q0, q1)
    assert float(track.sum()) == pytest.approx(float(oracle.exact_sum(dense)), rel=1e-12)
    assert bits([float(track.sum())]) == bits([float(track.sum())])
    assert float(track.max()) == np.max(dense) and float(track.min()) == np.min(dense)


# --------------------------------------------------------------------------------------------------------------------
# operators
# --------------------------------------------------------------------------------------------------------------------
OPS = [np.add, np.subtract, np.multiply, np.true_divide, np.minimum, np.maximum, np.equal, np.not_equal, np.less,
       np.less_equal, np.greater, np.greater_equal]


def _operands(rng, size):
    f = random_track(rng, size, 60, special=0.3)
    g = random_track(rng, size, 40, special=0.3)
    cuts = np.sort(rng.choice(np.arange(1, size), 15, replace=False))
    starts = np.concatenate([[0], cuts])
    ints = GenomicRunLengthArray.from_runs(starts, np.append(starts[1:], size), rng.integers(-3, 4, 16))
    bools = GenomicRunLengthArray.from_runs(starts, np.append(starts[1:], size),
                                            np.arange(16) % 2 == 0)
    return f, g, ints, bools


def test_every_operator_and_operand_kind_matches_numpy():
    rng = np.random.default_rng(2)
    size = 500
    f, g, ints, bools = _operands(rng, size)
    others = [g, ints, bools, 0, 3, -2, 2.5, -0.0, 0.0, math.inf, np.float32(1.5), np.int64(7), True]
    with np.errstate(all="ignore"):
        for op in OPS:
            for other in others:
                for args in ((f, other), (other, f)):
                    got = op(*args)
                    want = op(*[np.asarray(x) if isinstance(x, GenomicRunLengthArray) else x for x in args])
                    assert isinstance(got, GenomicRunLengthArray), (op, other)
                    if want.dtype == np.bool_:
                        assert got.dtype == torch.bool and np.array_equal(np.asarray(got), want), (op, other)
                    else:
                        assert isinstance(got, FloatRunLengthArray)
                        assert np.array_equal(bits(np.asarray(got)), bits(want)), (op, other)
                    _canonical(got)
        dense = np.asarray(f)
        assert np.array_equal(bits(np.asarray(-f)), bits(-dense))
        assert np.array_equal(np.asarray(np.logical_not(f)), np.logical_not(dense))
        assert np.array_equal(bits(np.asarray(f / ints)), bits(dense / np.asarray(ints)))
        assert np.array_equal(bits(np.asarray(2 / f)), bits(2 / dense))
    with pytest.raises(TypeError):
        ints / ints
    with pytest.raises(TypeError):
        ints / 2
    with pytest.raises(ValueError):
        f + random_track(rng, size + 1, 5)


def test_bitwise_equal_neighbours_merge_and_signed_zeros_do_not():
    t = FloatRunLengthArray.from_runs([0, 5, 10], [5, 10, 20], [1.0, -1.0, 2.0])
    z = t * 0.0
    assert z.values.cpu().tolist() == [0.0, -0.0, 0.0] and [math.copysign(1, v) for v in z.values.cpu().tolist()] == \
        [1, -1, 1]
    one = (t - t) + 1
    assert one.starts.cpu().tolist() == [0] and one.values.cpu().tolist() == [1.0]


def test_extract_and_bedgraph_rows_keep_every_bit():
    values = [-0.0, math.inf, math.nan, -math.inf, 0.0, 1e-320, -5.5]
    starts = list(range(0, 70, 10))
    t = FloatRunLengthArray.from_runs(starts, starts[1:] + [70], values)
    dense = np.repeat(np.array(values), 10)
    assert np.array_equal(bits(np.asarray(t)), bits(dense))
    assert np.array_equal(bits(t[[0, 15, 25, 69]].cpu().numpy()), bits(dense[[0, 15, 25, 69]]))
    assert bits([t[5]]) == bits([-0.0])
    bg = t.to_bedgraph("x")
    assert np.array_equal(bits(bg.value.cpu().numpy()), bits(values))
    genome = bnp.Genome.from_dict({"x": 30, "y": 40})
    data = GenomicArray._of(t, genome).get_data()
    assert data.value.dtype == torch.float64
    assert data.start.cpu().tolist() == [0, 10, 20, 0, 10, 20, 30]
    assert np.array_equal(bits(data.value.cpu().numpy()), bits(values))          # the NaN run ends at x's end
    windows = t[bnp.Interval(["x"] * 3, [0, 20, 40], [20, 40, 60])]
    assert np.array_equal(bits(windows.mean(axis=0).cpu().numpy() if hasattr(windows.mean(axis=0), "cpu")
                               else np.asarray(windows.mean(axis=0))), bits(dense[:60].reshape(3, 20).mean(axis=0)))


# --------------------------------------------------------------------------------------------------------------------
# workflows and the API
# --------------------------------------------------------------------------------------------------------------------
def test_the_guide_workflow():
    genome = bnp.Genome.from_file(_golden("small.chrom.sizes"))
    peaks = genome.read_intervals(_golden("small_peaks.narrowPeak"), buffer_type=bnp.io.BedBuffer)
    signal = genome.read_track(_golden("small_treat_pileup.bdg"))
    assert signal.dtype == torch.float64
    mx = signal[peaks].max(axis=-1).cpu().numpy()
    mean = signal[peaks].mean(axis=-1).cpu().numpy()
    assert mx.tolist() == GUIDE_MAX
    assert np.allclose(mean, GUIDE_MEAN, rtol=0, atol=5e-9)
    sizes = oracle.read_sizes(_golden("small.chrom.sizes"))
    dense = oracle.dense_track(oracle.read_bedgraph(_golden("small_treat_pileup.bdg")), sizes)
    intervals = oracle.read_bed(_golden("small_peaks.narrowPeak"))
    assert mean.tolist() == oracle.interval_mean(dense, intervals)
    assert len(peaks[signal[peaks].max(axis=-1) > 200]) == 9
    assert float(signal.sum()) == pytest.approx(float(sum(oracle.exact_sum(d) for d in dense.values())), rel=1e-15)
    assert "chr1" in repr(signal) and set(signal.to_dict()) == set(sizes)
    with pytest.raises(NotImplementedError):
        genome.read_track(_golden("small_treat_pileup.bdg"), stream=True)


def test_treat_control_chain_down_to_the_bed_bytes(tmp_path):
    rng = np.random.default_rng(9)
    sizes = {"chr1": 200_000, "chr2": 150_000, "chrM": 500}
    genome = bnp.Genome.from_dict(sizes)

    def write_track(path, scale):
        lines = []
        for name, size in sizes.items():
            cuts = np.sort(rng.choice(np.arange(1, size), min(size // 20, 4000), replace=False))
            edges = np.concatenate([[0], cuts, [size]])
            for a, b in zip(edges[:-1], edges[1:]):
                lines.append(f"{name}\t{a}\t{b}\t{rng.exponential(scale):.5f}\n")
        open(path, "w").write("".join(lines))

    treat_p, ctrl_p = str(tmp_path / "treat_pileup.bdg"), str(tmp_path / "control_lambda.bdg")
    write_track(treat_p, 6.0)
    write_track(ctrl_p, 2.0)
    treat, ctrl = genome.read_track(treat_p), genome.read_track(ctrl_p)
    ratio = (treat + 1) / (ctrl + 1)
    peaks = bnp.GenomicIntervals.from_track(ratio > 2).merged()
    out = str(tmp_path / "peaks.bed")
    bnp.open(out, "w", buffer_type=bnp.io.BedBuffer).write(peaks.get_data())
    t = oracle.dense_track(oracle.read_bedgraph(treat_p), sizes)
    c = oracle.dense_track(oracle.read_bedgraph(ctrl_p), sizes)
    want = []
    for name in sizes:
        r = (t[name] + 1) / (c[name] + 1)
        assert np.array_equal(bits(np.asarray(ratio[name])), bits(r))
        m = np.concatenate([[False], r > 2, [False]])
        d = np.flatnonzero(m[1:] != m[:-1])
        want += [f"{name}\t{a}\t{b}\n" for a, b in zip(d[0::2], d[1::2])]
    assert open(out).read() == "".join(want)


def test_the_pinned_integer_behaviours_hold():
    ev = torch.tensor([0, 5, 10], device="cuda")
    with pytest.raises(TypeError, match="integers or bool"):
        GenomicRunLengthArray(ev, torch.tensor([0.5, 1.0], device="cuda"))
    t = GenomicRunLengthArray.from_runs([0, 5], [5, 10], [1, 2])
    with pytest.raises(TypeError):
        t.astype(float)
    with pytest.raises(TypeError):
        GenomicRunLengthArray.from_runs([0, 5], [5, 10], [0.5, 1.0])
    assert isinstance(t + 0.5, np.ndarray) and np.array_equal(t + 0.5, np.asarray(t) + 0.5)
    assert isinstance(np.sqrt(t), np.ndarray)
    with pytest.raises(NotImplementedError):
        BdgBuffer.from_raw_buffer(bnp.as_encoded_array("x\t0\t1\t0.5\n"))
    with pytest.raises(TypeError):
        BdgBuffer.from_data(bnp.BedGraph(["x"], [0], [3], np.array([0.5])))


def test_dispatcher_ops_match_the_ctypes_ops():
    torch_ops.load()
    base, starts, lens = _device_text([b"1.5", b"-0", b"1e-320", b"x"])
    table = pow5_table(base.device)
    v1, s1 = torch.ops.bnpk.parse_float(base, starts, lens, 3, table)
    v2, s2 = ops.parse_float(base, starts, lens, 3, table)
    assert np.array_equal(bits(v1.cpu().numpy()), bits(v2.cpu().numpy()))
    assert ops.read_status(s1).column_fault() == (3, 3, nv.BAD_FLOAT) == ops.read_status(s2).column_fault()
    t = random_track(np.random.default_rng(1), 1000, 50)
    q0, q1 = torch.tensor([0, 10, 500], device="cuda"), torch.tensor([1000, 10, 900], device="cuda")
    for mode in (nv.RUNS_MAX, nv.RUNS_MIN, nv.RUNS_SUM, nv.RUNS_ANY):
        a = torch.ops.bnpk.track_f64_reduce(t._events, t.values, q0, q1, mode)
        b = ops.track_f64_reduce(t._events, t.values, q0, q1, mode)
        assert np.array_equal(bits(a.cpu().numpy()), bits(b.cpu().numpy()))
    s1, v1, n1 = torch.ops.bnpk.track_f64_combine(t._events, t.values, t._events, t.values, nv.OP_DIV)
    s2, v2, n2 = ops.track_f64_combine(t._events, t.values, t._events, t.values, nv.OP_DIV)
    n = int(n1.item())
    assert n == int(n2.item()) and torch.equal(s1[:n + 1], s2[:n + 1])
    assert np.array_equal(bits(v1[:n].cpu().numpy()), bits(v2[:n].cpu().numpy()))
    with pytest.raises(ValueError):
        ops.track_f64_combine(t._events, t.values, t._events, t.values, nv.OP_AND)
    with pytest.raises(TypeError):
        ops.parse_float(base, starts, lens, 3, table.to(torch.int32))
