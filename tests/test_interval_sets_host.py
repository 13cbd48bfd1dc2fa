"""Interval sets and track operators without a GPU: the NumPy oracle against the reference's goldens, the argument
checks of bnpk_runs_combine and bnpk_interval_intersect, their dispatcher schemas and their compiled code."""
import ctypes
import gzip
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

from bionumpy_b200 import _native as nv

import interval_sets_oracle as so
import pileup_oracle as po

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")

# tests/test_intervals.py of the reference
A = (["chr1"] * 3, np.array([10, 20, 30]), np.array([15, 29, 35]))
B = (["chr1"] * 3, np.array([10, 22, 29]), np.array([15, 28, 36]))
D = (["chr3", "chr2", "chr2", "chr1"], np.array([10, 15, 14, 12]), np.array([20, 22, 23, 24]))
SMALL = (["chr1"] * 4, np.array([2, 5, 10, 11]), np.array([5, 7, 12, 13]))
# tests/test_similarity_measures.py of the reference
SA = (["chr1", "chr2"], np.array([10, 20]), np.array([20, 30]))
SB = (["chr1", "chr2"], np.array([15, 15]), np.array([22, 25]))


def _bed(name):
    return po.parse_bed(gzip.open(os.path.join(GOLDEN, name)).read())


def test_count_overlap_golden():
    assert so.count_overlap(A, B) == 5 + 6 + 5


def test_intersect_golden():
    rows, stops = so.intersect(A, B)
    starts = np.concatenate([A[1], B[1]])[rows]
    assert starts.tolist() == [10, 22, 30] and stops.tolist() == [15, 28, 35]
    # the tie at 10: the sweep keeps b's row (the second of the stable order), with a's stop
    assert rows.tolist()[0] == 3


def test_unique_intersect_golden():
    assert so.unique_intersect(SMALL, (["chr1"], np.array([7]), np.array([11]))).tolist() == [2]


def test_sort_intervals_golden():
    assert so.sort_intervals(*D).tolist() == [3, 2, 1, 0]
    assert so.sort_intervals(*D, sort_order=["chr3", "chr1", "chr2"]).tolist() == [0, 3, 2, 1]
    with pytest.raises(KeyError):
        so.sort_intervals(*D, sort_order=["chr1", "chr2"])


def test_similarity_goldens():
    assert so.contingency_table(SA, SB, 150) == [[10, 10], [7, 123]]
    assert so.forbes({"chr1": 100, "chr2": 50}, SA, SB) == (150 * 10) / (20 * 17)
    assert so.jaccard({"chr1": 100, "chr2": 50}, SA, SB) == 10 / (12 + 15)
    a = (["chr1", "chr2"], np.array([10, 20]), np.array([20, 30]))
    b = (["chr2", "chr1"], np.array([15, 10]), np.array([25, 40]))
    assert so.forbes({"chr1": 100, "chr2": 200}, a, b) == 5.625


def test_global_intersect_cuts_at_chromosomes():
    a = (["chr1"], np.array([100]), np.array([200]))
    b = (["chr2"], np.array([10]), np.array([20]))
    rows, _ = so.global_intersect(b, a)
    assert rows.tolist() == []
    rows, stops = so.global_intersect(B, A)
    assert (rows.tolist(), stops.tolist()) == (so.intersect(A, B)[0].tolist(), so.intersect(A, B)[1].tolist())


def test_unique_intersect_example_count():
    """scripts/unique_intersect_example.py: ctcf peaks that meet a znf263 peak on hg38, every contig kept."""
    assert so.unique_intersect(_bed("ctcf.bed.gz"), _bed("znf263.bed.gz")).size == 3951


def test_dense_track_oracle():
    a = np.array([1, 1, 0, 0, 1], dtype=bool)
    b = np.array([0, 1, 1, 0, 0], dtype=bool)
    out, (s, e, v) = so.dense_op(np.bitwise_and, a, b)
    assert out.dtype == np.bool_ and (s.tolist(), e.tolist(), v.tolist()) == ([0, 1, 2], [1, 2, 5], [False, True, False])
    out, _ = so.dense_op(np.add, a, b)
    assert out.dtype == np.bool_ and out.tolist() == [True, True, True, False, True]
    out, _ = so.dense_op(np.add, np.array([2 ** 63 - 1], dtype=np.int64), 1)
    assert out.tolist() == [-2 ** 63]
    out, _ = so.dense_op(np.add, np.array([100], dtype=np.int8), np.array([100], dtype=np.int8))
    assert out.dtype == np.int64 and out.tolist() == [200]
    with pytest.raises(TypeError):
        so.dense_op(np.subtract, a, b)


def test_new_entry_points_bad_arguments():
    lib = nv.load_library()
    buf = ctypes.create_string_buffer(256)
    p = ctypes.cast(buf, ctypes.c_void_p)
    # a_starts, a_values, n_a, b_starts, b_values, n_b, op, out_starts, out_values, n_out, workspace, bytes, stream
    cb = [p, p, 2, p, p, 2, nv.OP_AND, p, p, p, p, 256, None]
    for i in (0, 1, 3, 4, 7, 8, 9, 10):
        args = list(cb)
        args[i] = None
        assert lib.bnpk_runs_combine(*args) == nv.E_BADARG, i
    for i, v in ((6, -1), (6, 14), (2, 0), (5, 0)):
        args = list(cb)
        args[i] = v
        assert lib.bnpk_runs_combine(*args) == nv.E_BADARG, (i, v)
    args = list(cb)
    args[11] = 8
    assert lib.bnpk_runs_combine(*args) == nv.E_WORKSPACE
    # start, stop, same_prev, n, out_rows, out_stops, n_out, overlap, workspace, workspace_bytes, stream
    it = [p, p, None, 4, p, p, p, None, p, 256, None]
    for i in (0, 1, 5, 6, 8):
        args = list(it)
        args[i] = None
        assert lib.bnpk_interval_intersect(*args) == nv.E_BADARG, i
    args = list(it)
    args[9] = 8
    assert lib.bnpk_interval_intersect(*args) == nv.E_WORKSPACE


def test_dispatcher_schemas():
    import torch
    lib = os.path.join(os.path.dirname(nv.LIB_PATH), "libbnpk_torch.so")
    if not os.path.exists(lib):
        pytest.skip("libbnpk_torch.so not built")
    torch.ops.load_library(lib)
    want = {
        "runs_combine": "bnpk::runs_combine(Tensor a_starts, Tensor a_values, Tensor b_starts, Tensor b_values, "
                        "int op) -> (Tensor, Tensor, Tensor)",
        "interval_intersect": "bnpk::interval_intersect(Tensor start, Tensor stop, Tensor? same_prev, bool rows) -> "
                              "(Tensor, Tensor, Tensor, Tensor)",
    }
    for name, schema in want.items():
        assert str(getattr(torch.ops.bnpk, name).default._schema) == schema


def test_new_kernels_are_sm90a_code_without_stack_or_spills():
    tool = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(tool):
        pytest.skip("cuobjdump not available")
    out = subprocess.run([tool, "-res-usage", nv.LIB_PATH], capture_output=True, text=True).stdout
    usage = {m.group(1): (int(m.group(2)), int(m.group(3)))
             for m in re.finditer(r"Function (\S+):\s*REG:(\d+) STACK:(\d+)", out)}
    names = ("runs_combine_kernel", "interval_intersect_kernel")
    found = {n: v for n, v in usage.items() if re.search("|".join(names), n)}
    assert len(found) == len(names), sorted(found)
    for name, (regs, stack) in found.items():
        assert stack == 0 and regs <= 128, (name, regs, stack)
    sass = subprocess.run([tool, "-sass", nv.LIB_PATH], capture_output=True, text=True).stdout
    for name in names:
        assert re.search(r"Function : \S*" + name, sass), name
    assert "arch = sm_90a" in sass
    for block in re.split(r"\n\s+Function : ", sass):
        if any(n in block.split("\n", 1)[0] for n in names):
            assert "STL" not in block and "LDL" not in block          # no local-memory spills


# --------------------------------------------------------------------------------------------------------------------
# the helpers of tests/test_gpu_track_ops.py
# --------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("m", [8, 16, 2040, 2047, 2048, 2049, 4096, 2048 * 40])
@pytest.mark.parametrize("side", ["a", "b", "ab"])
def test_event_tracks_placement(m, side):
    """The placed event is the m-th run start of a plain merge of both tracks, A before B at one position, and both
    tracks are well-formed runs of one size holding the event's values."""
    a, b, size, p = so.event_tracks([("ab", 1, 2), (side, 5, 6)], 1, m, after=9, seed=m)
    merged = sorted([(int(x), "A") for x in a[0]] + [(int(x), "B") for x in b[0]])
    assert merged[m] == (p, "A" if "a" in side else "B")
    if side == "ab":
        assert merged[m + 1] == (p, "B")
    assert len(merged) == m + len(side) + 9
    for starts, ends, values in (a, b):
        assert starts[0] == 0 and ends[-1] == size and np.all(starts[1:] == ends[:-1]) and np.all(ends > starts)
    da, db = po.dense_of(*a), po.dense_of(*b)
    assert (da[p], db[p]) == (5 if "a" in side else da[p - 1], 6 if "b" in side else db[p - 1])
    assert (da[p - 1], db[p - 1]) == (1, 2)


def test_event_tracks_exact_ends():
    for total in (2049, 2056, 4097):
        a, b, size, p = so.event_tracks([("a", 3, 0)], 0, total - 1, after=0, seed=total)
        assert a[0].size + b[0].size == total and a[0][-1] == p


def test_sweep_loop_matches_intersect():
    rng = np.random.default_rng(1)
    for n in (1, 2, 50, 700):
        a = (["chr1"] * n, rng.integers(0, 3 * n, n), None)
        a = (a[0], a[1], a[1] + rng.integers(0, 10, n))
        b = (["chr1"] * (n // 2 + 1), rng.integers(0, 3 * n, n // 2 + 1), None)
        b = (b[0], b[1], b[1] + rng.integers(0, 10, b[1].size))
        s, e = np.concatenate([a[1], b[1]]), np.concatenate([a[2], b[2]])
        order = np.argsort(s, kind="mergesort")
        rows, stops, over = so.sweep_loop(s[order], np.sort(e))
        want_rows, want_stops = so.intersect(a, b)
        assert order[rows].tolist() == want_rows.tolist() and stops.tolist() == want_stops.tolist()
        assert over == so.count_overlap(a, b)
    same = np.array([0, 1, 0, 1], dtype=np.uint8)
    rows, stops, over = so.sweep_loop(np.array([0, 1, 2, 3]), np.array([9, 9, 9, 9]), same)
    assert rows.tolist() == [1, 3] and stops.tolist() == [9, 9] and over == 8 + 6
    top = np.array([0, 1, 2], dtype=np.int64), np.array([2 ** 62, 2 ** 62 + 2 ** 61, 2 ** 62], dtype=np.int64)
    assert so.sweep_loop(*top)[2] == (2 ** 62 - 1) + (2 ** 62 + 2 ** 61 - 2) - 2 ** 64       # past 2^63: wraps


def test_mask_intersect_matches_intersect_on_merged_sets():
    rng = np.random.default_rng(2)
    for n in (1, 30, 400):
        sets = []
        for _ in range(2):
            s = np.sort(rng.integers(0, 10 * n, n))
            rows, stops = po.merge_intervals(s, s + rng.integers(1, 25, n))
            sets.append((["chr1"] * rows.size, s[rows], stops))
        a, b = sets
        rows, stops = so.intersect(a, b)
        starts = np.concatenate([a[1], b[1]])[rows]
        ws, we = so.mask_intersect(a, b)["chr1"]
        assert sorted(zip(starts.tolist(), stops.tolist())) == list(zip(ws.tolist(), we.tolist()))
        assert int((we - ws).sum()) == so.count_overlap(a, b)
