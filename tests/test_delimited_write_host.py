"""BED and bedGraph writing and track rows without a GPU: the oracle against the reference's goldens, the argument
checks of bnpk_runs_to_intervals, bnpk_delimited_offsets and bnpk_delimited_format, and their compiled code."""
import ctypes
import gzip
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

from bionumpy_b200 import _native as nv

import delimited_write_oracle as wo
import interval_oracle as io_

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _golden(name):
    path = os.path.join(GOLDEN, name)
    return gzip.open(path).read() if name.endswith(".gz") else open(path, "rb").read()


def test_small_interval_bed_writes_back_byte_for_byte():
    text = _golden("small_interval.bed")
    chrom, start, stop = io_.parse_delimited(text, io_.BED)[1]
    assert wo.dump_lines(wo.bed_columns(chrom, start, stop)) == text


def test_ctcf_as_bed3_writes_its_first_three_columns():
    text = _golden("ctcf.bed.gz")
    chrom, start, stop = io_.parse_delimited(text, io_.BED)[1]
    cut = b"".join(b"\t".join(line.split(b"\t")[:3]) + b"\n" for line in text.splitlines())
    assert wo.dump_lines(wo.bed_columns(chrom, start, stop)) == cut


def test_alignments_as_bed6_write_dot_scores_as_zero():
    text = _golden("alignments.bed")
    cols = io_.parse_delimited(text, io_.BED6)[1]
    kinds = ("text", "int", "int", "text", "int", "strand")
    out = wo.dump_lines(list(zip(kinds, cols)))
    want = b"".join(b"\t".join(f[:4] + [b"0" if f[4] == b"." else f[4]] + f[5:6]) + b"\n"
                    for f in (line.split(b"\t") for line in text.splitlines()))
    assert out == want and b"\t.\t+" not in out and out.count(b"\t0\t") == text.count(b"\t.\t.\t")


def test_oracle_integers_and_runs():
    assert wo.ints_to_strings([0, -9, 10, -(1 << 63), (1 << 63) - 1]) == \
        [b"0", b"-9", b"10", b"-9223372036854775808", b"9223372036854775807"]
    names, s, e = wo.nonzero_intervals({"a": [0, 1, 2, 0], "b": [3, 3], "c": []})
    assert names == ["a", "b"] and s.tolist() == [1, 0] and e.tolist() == [3, 2]
    names, s, e, v = wo.bedgraph_rows({"a": [0, 1, 1], "b": [5]})
    assert names == ["a", "a", "b"] and s.tolist() == [0, 1, 0] and e.tolist() == [1, 3, 1] and v.tolist() == [0, 1, 5]
    dense = wo.dense_of_rows(names, s, e, v, {"a": 3, "b": 1})
    assert dense["a"].tolist() == [0, 1, 1] and dense["b"].tolist() == [5]


# --------------------------------------------------------------------------------------------------------------------
# argument errors: refused before any device work, so no GPU is needed
# --------------------------------------------------------------------------------------------------------------------
def _err(rc):
    assert rc == nv.E_BADARG, rc
    return nv.load_library().bnpk_last_error().decode()


def test_runs_to_intervals_argument_errors():
    lib = nv.load_library()
    fake = ctypes.c_void_p(16)
    args = lambda **kw: [kw.get(k, d) for k, d in (
        ("starts", fake), ("values", fake), ("n", 4), ("ends", fake), ("c", 2), ("mode", nv.RUNS_TO_NONZERO),
        ("contig", fake), ("start", fake), ("stop", fake), ("value", None), ("n_out", fake), ("ws", fake),
        ("ws_bytes", 1 << 20), ("stream", None))]
    assert "mode" in _err(lib.bnpk_runs_to_intervals(*args(mode=7)))
    assert "n_out" in _err(lib.bnpk_runs_to_intervals(*args(n_out=None)))
    assert "n_contigs" in _err(lib.bnpk_runs_to_intervals(*args(c=0)))
    assert "required" in _err(lib.bnpk_runs_to_intervals(*args(mode=nv.RUNS_TO_ALL)))   # ALL writes values
    assert "required" in _err(lib.bnpk_runs_to_intervals(*args(ends=None)))


def _columns(*cols):
    arr = (nv.OutColumn * max(len(cols), 1))()
    for i, c in enumerate(cols):
        arr[i] = c
    return ctypes.cast(arr, ctypes.c_void_p)


def test_delimited_argument_errors():
    lib = nv.load_library()
    text = nv.OutColumn(nv.COL_TEXT, 16, 8, 16, 16)
    ints = nv.OutColumn(nv.COL_INT, 16, 0, None, None)
    ws = ctypes.c_void_p(16)
    assert "columns" in _err(lib.bnpk_delimited_offsets(_columns(), 0, 1, ws, ws, ws, 1 << 20, None))
    assert "columns" in _err(lib.bnpk_delimited_offsets(_columns(*[ints] * 9), 9, 1, ws, ws, ws, 1 << 20, None))
    for kind in (nv.COL_SKIP, nv.COL_INT_OR_DOT, 99):
        bad = nv.OutColumn(kind, 16, 0, None, None)
        assert "BNPK_COL" in _err(lib.bnpk_delimited_offsets(_columns(text, bad), 2, 1, ws, ws, ws, 1 << 20, None))
    no_lens = nv.OutColumn(nv.COL_TEXT, 16, 8, 16, None)
    assert "misses" in _err(lib.bnpk_delimited_offsets(_columns(no_lens), 1, 1, ws, ws, ws, 1 << 20, None))
    assert "out_offsets" in _err(lib.bnpk_delimited_offsets(_columns(ints), 1, 1, None, ws, ws, 1 << 20, None))
    assert "status" in _err(lib.bnpk_delimited_offsets(_columns(ints), 1, 1, ws, None, ws, 1 << 20, None))
    assert "out_begin" in _err(lib.bnpk_delimited_format(_columns(ints), 1, 1, ws, 5, 4, ws, None))
    assert "out_begin" in _err(lib.bnpk_delimited_format(_columns(ints), 1, 1, ws, -1, 4, ws, None))
    assert "NULL" in _err(lib.bnpk_delimited_format(_columns(ints), 1, 1, ws, 0, 4, None, None))
    assert "offsets" in _err(lib.bnpk_delimited_format(_columns(ints), 1, 1, None, 0, 4, ws, None))
    assert lib.bnpk_delimited_format(_columns(ints), 1, 1, ws, 3, 3, None, None) == 0          # an empty range


def test_dispatcher_schemas():
    import torch
    from bionumpy_b200 import torch_ops
    ops = torch_ops.load()
    for name in ("runs_to_intervals", "delimited_offsets", "delimited_format"):
        assert hasattr(ops, name), name
    assert "int[] kinds" in str(torch._C._get_schema("bnpk::delimited_format", ""))


def test_new_kernels_are_sm90a_code_without_stack_or_spills():
    tool = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(tool):
        pytest.skip("cuobjdump not available")
    out = subprocess.run([tool, "-res-usage", nv.LIB_PATH], capture_output=True, text=True).stdout
    usage = {m.group(1): (int(m.group(2)), int(m.group(3)))
             for m in re.finditer(r"Function (\S+):\s*REG:(\d+) STACK:(\d+)", out)}
    names = ("runs_to_intervals_kernel", "delimited_offsets_kernel", "delimited_text_kernel")
    found = {n: v for n, v in usage.items() if re.search("|".join(names), n)}
    assert len(found) == len(names), sorted(found)
    for name, (regs, stack) in found.items():
        assert stack == 0 and regs <= 64, (name, regs, stack)
    sass = subprocess.run([tool, "-sass", nv.LIB_PATH], capture_output=True, text=True).stdout
    assert "arch = sm_90a" in sass
    for block in re.split(r"\n\s+Function : ", sass):
        if any(n in block.split("\n", 1)[0] for n in names):
            assert "STL" not in block and "LDL" not in block          # no local-memory spills
