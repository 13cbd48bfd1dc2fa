"""Pileups without a GPU: the NumPy oracle against the reference's goldens, the argument checks of the new C entry
points, the missing-GPU error, the dispatcher schemas and the compiled code of the pileup kernels."""
import ctypes
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

from bionumpy_b200 import _native as nv

import pileup_oracle as po

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")

# tests/test_pileup.py of the reference, at size 12
PILEUP_LISTS = [([2, 3, 5, 7], [4, 6, 8, 10]), ([2, 3, 3, 5, 7], [4, 6, 8, 8, 10]), ([2, 3, 3, 5, 7], [4, 6, 7, 8, 10])]
# tests/test_intervals.py complicated_intervals, at size 20
COMPLICATED = [([2, 5, 10, 11], [5, 7, 12, 13]), ([0, 11], [5, 13]), ([0, 11], [5, 20]), ([0, 11, 20], [5, 18, 20])]


def test_pileup_docstring():
    p = po.dense_pileup([3, 5, 10], [8, 7, 12], 20)
    assert " ".join(map(str, p)) == "0 0 0 1 1 2 2 1 0 0 1 1 0 0 0 0 0 0 0 0"
    s, e, v = po.runs_of(p)
    es, ee, ev = po.event_runs([3, 5, 10], [8, 7, 12], 20)
    assert s.tolist() == es.tolist() and e.tolist() == ee.tolist() and v.tolist() == ev.tolist()


def test_boolean_mask_docstring():
    mask = po.dense_mask([3, 5, 10], [8, 7, 12], 20)
    assert " ".join(map(str, mask.astype(int))) == "0 0 0 1 1 1 1 1 0 0 1 1 0 0 0 0 0 0 0 0"
    assert " ".join(map(str, (~mask).astype(int))) == "1 1 1 0 0 0 0 0 1 1 0 0 1 1 1 1 1 1 1 1"
    other = po.dense_mask([9], [15], 20)
    assert " ".join(map(str, (mask & other).astype(int))) == "0 0 0 0 0 0 0 0 0 0 1 1 0 0 0 0 0 0 0 0"
    assert " ".join(map(str, (mask | other).astype(int))) == "0 0 0 1 1 1 1 1 0 1 1 1 1 1 1 0 0 0 0 0"
    assert other[[3, 5, 10]].tolist() == [False, False, True]
    s, e, v = po.event_runs([3, 5, 10], [8, 7, 12], 20, any_mode=True)
    assert (s.tolist(), e.tolist(), v.tolist()) == ([0, 3, 8, 10, 12], [3, 8, 10, 12, 20], [False, True, False, True, False])


@pytest.mark.parametrize("starts,stops", PILEUP_LISTS)
def test_pileup_lists(starts, stops):
    raw = np.zeros(12, dtype=int)
    for a, b in zip(starts, stops):
        raw[a:b] += 1
    assert po.dense_pileup(starts, stops, 12).tolist() == raw.tolist()
    s, e, v = po.event_runs(starts, stops, 12)
    assert np.repeat(v, e - s).tolist() == raw.tolist()


@pytest.mark.parametrize("starts,stops", COMPLICATED)
def test_complicated_masks(starts, stops):
    true = np.zeros(20, dtype=bool)
    for a, b in zip(starts, stops):
        true[a:b] |= True
    s, e, v = po.event_runs(starts, stops, 20, any_mode=True)
    assert np.repeat(v, e - s).tolist() == true.tolist()
    assert np.all(v[1:] != v[:-1]) and s[0] == 0 and e[-1] == 20


def test_merge_fixture():
    """tests/test_util.py::test_merged_intervals."""
    rows, stops = po.merge_intervals([1, 2, 2, 10, 12, 20], [5, 3, 4, 15, 17, 25])
    assert np.array([1, 2, 2, 10, 12, 20])[rows].tolist() == [1, 10, 20] and stops.tolist() == [5, 17, 25]
    with pytest.raises(AssertionError, match="sorted on start position"):
        po.merge_intervals([1, 2, 10, 2], [5, 4, 15, 3])
    rows, stops = po.merge_intervals([0, 5, 5, 9], [5, 5, 7, 9])       # touching and zero-length rows
    assert rows.tolist() == [0, 3] and stops.tolist() == [7, 9]
    rows, stops = po.merge_intervals([0, 8], [5, 9], distance=3)
    assert rows.tolist() == [0] and stops.tolist() == [9]
    rows, stops = po.merge_by_chromosome(["chr1", "chr1", "chr2"], np.array([0, 3, 1]), np.array([5, 6, 2]))
    assert rows.tolist() == [0, 2] and stops.tolist() == [6, 2]


def test_genome_docstrings():
    """genome.py from_dict / from_file / get_intervals docstrings."""
    names, offsets, size = po.genome_layout({"chr1": 20, "chr2": 10})
    assert names == ["chr1", "chr2"] and offsets == {"chr1": 0, "chr2": 20} and size == 30
    keep, gs, ge = po.genome_intervals({"chr1": 20, "chr2": 10}, ["chr1", "chr1", "chr2"], [0, 10, 0], [5, 15, 5])
    assert keep.tolist() == [0, 1, 2] and gs.tolist() == [0, 10, 20] and ge.tolist() == [5, 15, 25]
    sizes = po.read_sizes(open(os.path.join(GOLDEN, "hg38.chrom.sizes")).read())
    names, _, _ = po.genome_layout(sizes)
    assert len(sizes) == 455 and names[:10] == ["chr%d" % i for i in range(1, 11)]
    assert sum("_" in n for n in sizes) == 455 - len(names)


def test_genome_repr_without_gpu():
    from bionumpy_b200.genomic_data import Genome
    assert repr(Genome.from_dict({"chr1": 1000, "chr2": 2000})) == "Genome(['chr1', 'chr2'])"
    g = Genome.from_file(os.path.join(GOLDEN, "hg38.chrom.sizes"))
    assert repr(g) == "Genome(['chr1', 'chr2', 'chr3', 'chr4', 'chr5', 'chr6', 'chr7', 'chr8', 'chr9', 'chr10', '...'])"
    assert "chr1_KI270706v1_random" not in g.chrom_sizes and g.size == sum(g.chrom_sizes.values())
    assert Genome.from_file(os.path.join(GOLDEN, "small_genome.fa")).chrom_sizes == \
        {k: v["rlen"] for k, v in _fai(os.path.join(GOLDEN, "small_genome.fa.fai")).items()}


def _fai(path):
    out = {}
    for line in open(path):
        f = line.split("\t")
        out[f[0]] = {"rlen": int(f[1])}
    return out


def test_oracle_event_runs_match_dense_runs():
    rng = np.random.default_rng(3)
    for size in (1, 2, 17, 300):
        for n in (0, 1, 2, 50):
            a = rng.integers(0, size + 1, n)
            b = np.minimum(a + rng.integers(0, 40, n), size)
            for any_mode in (False, True):
                dense = po.dense_pileup(a, b, size)
                dense = dense > 0 if any_mode else dense
                want = po.runs_of(dense)
                got = po.event_runs(a, b, size, any_mode)
                assert all(x.tolist() == y.tolist() for x, y in zip(want, got)), (size, n, any_mode)


def _lib():
    return nv.load_library()


def test_new_entry_points_bad_arguments():
    lib = _lib()
    buf = ctypes.create_string_buffer(256)
    p = ctypes.cast(buf, ctypes.c_void_p)
    # start, stop, ids, contig_offset, contig_len, n_contigs, size, n_rows, keys, g_start, g_stop, status, stream
    ev = [p, p, None, None, None, 0, 10, 1, p, None, None, p, None]
    for i in (0, 1, 11):
        args = list(ev)
        args[i] = None
        assert lib.bnpk_interval_events(*args) == nv.E_BADARG, i
    for i in (3, 4):                                  # ids without a contig column
        args = list(ev)
        args[2] = p
        args[3] = args[4] = p
        args[i] = None
        assert lib.bnpk_interval_events(*args) == nv.E_BADARG, i
    for size in (-1, 1 << 59):
        args = list(ev)
        args[6] = size
        assert lib.bnpk_interval_events(*args) == nv.E_BADARG
    args = list(ev)
    args[7] = 0
    assert lib.bnpk_interval_events(*args) == 0
    # keys, n_keys, size, mode, run_starts, run_values, n_runs, workspace, workspace_bytes, stream
    runs = [p, 4, 10, nv.PILEUP_COUNT, p, p, p, p, 256, None]
    for i in (0, 4, 5, 6, 7):
        args = list(runs)
        args[i] = None
        assert lib.bnpk_pileup_runs(*args) == nv.E_BADARG, i
    for i, v in ((3, 2), (3, -1), (2, -1), (2, 1 << 59)):
        args = list(runs)
        args[i] = v
        assert lib.bnpk_pileup_runs(*args) == nv.E_BADARG, (i, v)
    args = list(runs)
    args[8] = 8
    assert lib.bnpk_pileup_runs(*args) == nv.E_WORKSPACE
    # run_starts, values, n_runs, q_start, q_stop, n_q, mode, out, scratch, workspace, workspace_bytes, stream
    red = [p, p, 2, p, p, 1, nv.RUNS_MAX, p, p, p, 256, None]
    for i in (0, 1, 3, 4, 7, 8, 9):
        args = list(red)
        args[i] = None
        assert lib.bnpk_runs_reduce(*args) == nv.E_BADARG, i
    for i, v in ((6, 4), (6, -1), (2, 0)):
        args = list(red)
        args[i] = v
        assert lib.bnpk_runs_reduce(*args) == nv.E_BADARG, (i, v)
    args = list(red)
    args[5] = 0
    assert lib.bnpk_runs_reduce(*args) == 0
    # run_starts, values, n_runs, q_start, n_q, out_offsets, out, stream
    ext = [p, p, 2, p, 1, p, p, None]
    for i, v in ((0, None), (1, None), (2, 0), (3, None), (5, None), (6, None)):
        args = list(ext)
        args[i] = v
        assert lib.bnpk_runs_extract(*args) == nv.E_BADARG, i
    # start, stop, same_prev, n_rows, distance, out_rows, out_stops, n_out, status, workspace, workspace_bytes, stream
    mg = [p, p, None, 4, 0, p, p, p, p, p, 256, None]
    for i in (0, 1, 5, 6, 7, 8, 9):
        args = list(mg)
        args[i] = None
        assert lib.bnpk_interval_merge(*args) == nv.E_BADARG, i
    for d in (-1, 1 << 59):
        args = list(mg)
        args[4] = d
        assert lib.bnpk_interval_merge(*args) == nv.E_BADARG
    args = list(mg)
    args[10] = 8
    assert lib.bnpk_interval_merge(*args) == nv.E_WORKSPACE
    # base, base_bytes, starts, lens, n_rows, flag, stream
    eq = [p, 8, p, p, 1, p, None]
    for i in (0, 2, 3, 5):
        args = list(eq)
        args[i] = None
        assert lib.bnpk_rows_equal_prev(*args) == nv.E_BADARG, i
    args = list(eq)
    args[4] = 0
    assert lib.bnpk_rows_equal_prev(*args) == 0


def test_pileup_fails_loudly_without_gpu():
    import torch
    if torch.cuda.is_available():
        pytest.skip("a CUDA device is present")
    import bionumpy_b200 as bnp
    iv = bnp.Interval.__new__(bnp.Interval)
    iv.__dict__.update({"_buffer": None, "_values": {"chromosome": None, "start": [1], "stop": [2]}})
    for fn in (bnp.arithmetics.get_pileup, bnp.arithmetics.get_boolean_mask):
        with pytest.raises(nv.NativeLibraryError):
            fn(iv, 10)


def test_dispatcher_schemas():
    import torch
    lib = os.path.join(os.path.dirname(nv.LIB_PATH), "libbnpk_torch.so")
    if not os.path.exists(lib):
        pytest.skip("libbnpk_torch.so not built")
    torch.ops.load_library(lib)
    want = {
        "interval_events": "bnpk::interval_events(Tensor start, Tensor stop, Tensor? ids, Tensor? contig_offset, "
                           "Tensor? contig_len, int size) -> (Tensor, Tensor)",
        "pileup_runs": "bnpk::pileup_runs(Tensor keys, int size, int mode) -> (Tensor, Tensor, Tensor)",
        "runs_reduce": "bnpk::runs_reduce(Tensor run_starts, Tensor values, Tensor q_start, Tensor q_stop, int mode) "
                       "-> Tensor",
        "runs_extract": "bnpk::runs_extract(Tensor run_starts, Tensor values, Tensor q_start, Tensor offsets, "
                        "int total) -> Tensor",
        "interval_merge": "bnpk::interval_merge(Tensor start, Tensor stop, Tensor? same_prev, int distance) -> "
                          "(Tensor, Tensor, Tensor, Tensor)",
        "rows_equal_prev": "bnpk::rows_equal_prev(Tensor base, Tensor starts, Tensor lens) -> Tensor",
    }
    for name, schema in want.items():
        assert str(getattr(torch.ops.bnpk, name).default._schema) == schema


def test_pileup_kernels_are_sm90a_code_without_stack():
    tool = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(tool):
        pytest.skip("cuobjdump not available")
    out = subprocess.run([tool, "-res-usage", nv.LIB_PATH], capture_output=True, text=True).stdout
    usage = {m.group(1): (int(m.group(2)), int(m.group(3)))
             for m in re.finditer(r"Function (\S+):\s*REG:(\d+) STACK:(\d+)", out)}
    names = ("interval_events_kernel", "pileup_runs_kernel", "runs_locate_kernel", "count_scan_kernel",
             "runs_reduce_kernel", "runs_extract_kernel", "interval_merge_kernel", "rows_equal_prev_kernel")
    found = {n: v for n, v in usage.items() if re.search("|".join(names), n)}
    assert len(found) == len(names), sorted(found)
    for name, (regs, stack) in found.items():
        assert stack == 0 and regs <= 128, (name, regs, stack)
    # the row kernels are unchanged
    golden = open(os.path.join(GOLDEN, "rows_kernel_res_usage.txt")).read()
    rows = [line.split() for line in golden.splitlines() if line.strip()]
    assert rows
    for name, regs_stack in rows:
        regs, stack = regs_stack.split("/")
        assert usage.get(name) == (int(regs), int(stack)), name


def test_run_length_values_must_not_be_floating_point():
    import torch
    from bionumpy_b200.arithmetics import GenomicRunLengthArray
    events = torch.tensor([0, 3, 5])
    with pytest.raises(TypeError, match="integers or bool"):
        GenomicRunLengthArray(events, torch.tensor([0.5, 1.0]))
    assert GenomicRunLengthArray(events, torch.tensor([1, 0]), 5).dtype == torch.int64


DTYPES = [np.int64, np.int32, np.int16, np.int8, np.uint8, np.bool_]
HOWS = ("max", "min", "sum", "mean", "any")


def _same(got, want):
    got, want = np.asarray(got), np.asarray(want)
    assert got.shape == want.shape
    if got.dtype.kind == "f" or want.dtype.kind == "f":
        np.testing.assert_array_equal(got.astype(np.float64), want.astype(np.float64))
    else:
        assert got.tolist() == want.tolist()


def _queries(rng, size, n):
    """Random queries reaching 3 positions past both ends, reversed, empty and duplicated ones included."""
    a = rng.integers(-3, size + 4, n)
    b = np.where(rng.random(n) < 0.8, a + rng.integers(0, size // 2 + 3, n), rng.integers(-3, size + 4, n))
    a[: n // 8], b[: n // 8] = a[n // 8: 2 * (n // 8)], b[n // 8: 2 * (n // 8)]
    return a, b


@pytest.mark.parametrize("dtype", DTYPES)
def test_dense_of_inverts_runs_of(dtype):
    rng = np.random.default_rng(30)
    for size in (0, 1, 2, 7, 100):
        dense = po.random_dense(rng, size, dtype)
        s, e, v = po.runs_of(dense)
        back = po.dense_of(s, e, v)
        assert back.dtype == dense.dtype and back.tolist() == dense.tolist()
        assert np.all(v[1:] != v[:-1]) and (size == 0 or (s[0] == 0 and e[-1] == size))
        again = po.runs_of(back)
        assert all(x.tolist() == y.tolist() for x, y in zip((s, e, v), again))
    assert po.dense_of([0, 2, 5], [2, 5, 6], [7, -1, 3], np.int8).tolist() == [7, 7, -1, -1, -1, 3]


@pytest.mark.parametrize("dtype", DTYPES)
def test_dense_reducer_against_loop_and_runs(dtype):
    """reduce_dense equals a plain loop over the positions of every query and, on the clipped queries, reduce_runs
    (which works from the runs), for every dtype with its extreme values, empty rows following RaggedArray."""
    rng = np.random.default_rng(31)
    for size in (0, 1, 2, 5, 40, 300):
        dense = po.random_dense(rng, size, dtype)
        a, b = _queries(rng, size, 200)
        a = np.concatenate([a, [0, size, -5, size + 5, 3, 0]])
        b = np.concatenate([b, [size, size, -1, size + 9, 1, 0]])
        for how in HOWS:
            want = po.reduce_dense(dense, a, b, how)
            _same(want, po.reduce_loop(dense, a, b, how))
            if how in ("max", "min"):
                assert want.dtype == dense.dtype
            if size == 0 or how == "mean":
                continue
            s, e, v = po.runs_of(dense)
            ca, cb = po.clip_queries(a, b, size)
            runs = po.reduce_runs(s, e, v, ca, cb, how)
            full = cb > ca
            _same(want[full], runs[full].astype(want.dtype))
            if dtype == np.int64 or how in ("sum", "any"):
                _same(want, runs.astype(want.dtype))


def test_dense_reducer_empty_rows():
    dense = np.array([5, -3, 7], dtype=np.int16)
    a, b = np.array([1, 2, 9, -4, 2]), np.array([1, 0, 12, -1, 3])
    info = np.iinfo(np.int16)
    assert po.reduce_dense(dense, a, b, "max").tolist() == [info.min] * 4 + [7]
    assert po.reduce_dense(dense, a, b, "min").tolist() == [info.max] * 4 + [7]
    assert po.reduce_dense(dense, a, b, "sum").tolist() == [0, 0, 0, 0, 7]
    assert np.isnan(po.reduce_dense(dense, a, b, "mean")[:4]).all()
    assert po.reduce_dense(dense, a, b, "any").tolist() == [False] * 4 + [True]
    flags = np.array([True, False])
    assert po.reduce_dense(flags, [0, 1, 1, 2], [0, 2, 1, 2], "max").tolist() == [False, False, False, False]
    assert po.reduce_dense(flags, [0, 1, 1, 2], [0, 2, 1, 2], "min").tolist() == [True, False, True, True]
    assert po.reduce_dense(flags, [0], [2], "max").tolist() == [True]


def test_dense_reducer_wrapping_sums():
    """Sums near and past 2^63 wrap modulo 2^64, as the kernels' uint64 arithmetic does: checked against exact Python
    integers.  The mean is exact only where mean_is_exact says so."""
    rng = np.random.default_rng(32)
    lens = rng.integers(1, 50, 40)
    vals = (1 << 62) + rng.integers(-1000, 1000, 40)
    vals[::7] = -(1 << 62) - rng.integers(0, 1000, vals[::7].size)
    dense = np.repeat(vals.astype(np.int64), lens)
    a = rng.integers(0, dense.size, 300)
    b = a + rng.integers(0, dense.size, 300)
    got = po.reduce_dense(dense, a, b, "sum")
    ca, cb = po.clip_queries(a, b, dense.size)
    for g, s, e in zip(got, ca, cb):
        exact = sum(int(v) for v in dense[s:e])
        assert int(g) % 2 ** 64 == exact % 2 ** 64
    assert (np.abs([sum(int(v) for v in dense[s:e]) for s, e in zip(ca, cb)]) >= 2 ** 63).any()   # some do wrap
    _same(po.reduce_dense(dense, a, b, "mean"), po.reduce_loop(dense, a, b, "mean"))
    exact = po.mean_is_exact(dense, a, b)
    assert exact[cb - ca <= 0].all() and not exact[cb - ca > 2].any()
    small = np.arange(-50, 50, dtype=np.int64)
    assert po.mean_is_exact(small, [0, 10], [100, 90]).all()
    assert po.reduce_dense(small, [0, 10], [100, 90], "mean").tolist() == [-0.5, -0.5]
