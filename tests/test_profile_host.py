"""Track profiles without a GPU: tests/profile_oracle.py on hand-worked locations, windows, extensions and column
sums, the C-ABI constants and dispatcher schemas of K18, the .narrowPeak suffix mapping, and the machine code of the
new kernels."""
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

import profile_oracle as oracle
from bionumpy_b200 import _native as nv

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
KERNELS = ("column_sum_kernel", "column_fold_kernel")


def test_minus_interval_locations_and_windows():
    assert oracle.location(10, 20, "-", "start") == 19
    assert oracle.location(10, 20, "-", "stop") == 10
    assert oracle.location(10, 20, "+", "start") == 10
    assert oracle.location(10, 20, "+", "stop") == 19
    assert oracle.location(10, 20, ".", "stop") == 19
    assert oracle.location(10, 20, None, "stop") == 19
    assert oracle.location(10, 21, "-", "center") == 15
    assert oracle.window(19, 100, flank=5) == (14, 25)
    assert oracle.window(19, 100, window_size=10) == (14, 24)
    assert oracle.window(19, 100, window_size=11) == (14, 25)


def test_windows_at_both_contig_ends_are_clipped():
    assert oracle.window(2, 100, flank=5) == (0, 8)
    assert oracle.window(0, 100, flank=5) == (0, 6)
    assert oracle.window(97, 100, flank=5) == (92, 100)
    assert oracle.window(99, 100, flank=5) == (94, 100)


def test_extension_along_the_strand():
    assert oracle.extended(10, 20, "+", 50, 100) == (10, 60)
    assert oracle.extended(10, 20, ".", 50, 100) == (10, 60)
    assert oracle.extended(10, 20, None, 50, 100) == (10, 60)
    assert oracle.extended(10, 20, "-", 50, 100) == (0, 20)
    assert oracle.extended(70, 90, "+", 50, 100) == (70, 100)


def test_rows_read_back_to_front_on_reversed_rows():
    track = np.arange(20)
    m = oracle.rows(track, [0, 5], 4, [False, True])
    assert m.tolist() == [[0, 1, 2, 3], [8, 7, 6, 5]]


def test_blocked_column_sum_order():
    rng = np.random.default_rng(0)
    m = rng.standard_normal((oracle.BLOCK_ROWS, 7)) * 10.0 ** rng.integers(-20, 20, (oracle.BLOCK_ROWS, 7))
    assert np.array_equal(oracle.column_sum(m), m.sum(axis=0))       # one block: NumPy's row-by-row sum from +0.0
    big = np.vstack([m, m[:3]])
    want = np.zeros(7) + m.sum(axis=0)
    want = want + (np.zeros(7) + m[0] + m[1] + m[2])
    assert np.array_equal(oracle.column_sum(big), want)
    # every partial starts from +0.0, so an all -0.0 column sums to +0.0
    neg = np.full((3, 1), -0.0)
    assert np.signbit(neg.sum(axis=0)[0]) == np.signbit(oracle.column_sum(neg)[0]) == False  # noqa: E712
    wrap = np.array([[2 ** 62], [2 ** 62], [2 ** 62]], dtype=np.int64)
    assert oracle.column_sum(wrap).tolist() == [-(2 ** 62)]


def test_oracle_reads_narrowpeak():
    rows = oracle.read_narrowpeak(os.path.join(GOLDEN, "small_peaks.narrowPeak"))
    assert rows[0] == ("chr1", 482, 790, "small_peak_1", 1521, ".", 10.8571, 152.18, 150.464, 157)
    assert len(rows) == 13
    ctcf = oracle.read_narrowpeak(os.path.join(GOLDEN, "ctcf_chr21-22.bed.gz"))
    assert ctcf[0][7] == -1.0 and ctcf[0][9] == 135


def test_header_constants():
    text = open(os.path.join(ROOT, "include", "bnpk.h")).read()
    m = re.search(r"#define\s+BNPK_COLUMN_BLOCK_ROWS\s+(\d+)", text)
    assert m and int(m.group(1)) == nv.COLUMN_BLOCK_ROWS == oracle.BLOCK_ROWS
    assert "#define BNPK_ABI_VERSION 3" in text
    for name in ("bnpk_runs_column_sum", "bnpk_track_f64_column_sum"):
        assert name in text and name in nv.SIGNATURES


def test_library_exports_the_new_entry_points():
    if not os.path.exists(nv.LIB_PATH):
        pytest.skip("libbnpk.so not built")
    lib = nv.load_library()
    for name in ("bnpk_runs_column_sum", "bnpk_track_f64_column_sum"):
        assert hasattr(lib, name)


def test_bad_arguments_are_refused_before_device_work():
    if not os.path.exists(nv.LIB_PATH):
        pytest.skip("libbnpk.so not built")
    lib = nv.load_library()
    p = 16          # never dereferenced: every call below is refused first
    for fn in (lib.bnpk_runs_column_sum, lib.bnpk_track_f64_column_sum):
        assert fn(p, p, 1, p, None, 1, -1, p, p, None) == nv.E_BADARG
        assert fn(p, p, 1, p, None, 1, 1 << 31, p, p, None) == nv.E_BADARG
        assert fn(None, p, 1, p, None, 1, 4, p, p, None) == nv.E_BADARG
        assert fn(p, p, 0, p, None, 1, 4, p, p, None) == nv.E_BADARG
        assert fn(p, p, 1, p, None, 1, 4, None, p, None) == nv.E_BADARG
        assert fn(p, p, 1, None, None, 1, 4, p, p, None) == nv.E_BADARG
        assert fn(p, p, 1, p, None, 1, 4, p, None, None) == nv.E_BADARG
        assert fn(p, p, 1, None, None, 0, 0, None, None, None) == 0          # nothing to write


def test_dispatcher_schemas():
    import torch
    lib = os.path.join(os.path.dirname(nv.LIB_PATH), "libbnpk_torch.so")
    if not os.path.exists(lib):
        pytest.skip("libbnpk_torch.so not built")
    torch.ops.load_library(lib)
    for name in ("runs_column_sum", "track_f64_column_sum"):
        assert str(getattr(torch.ops.bnpk, name).default._schema) == (
            f"bnpk::{name}(Tensor run_starts, Tensor values, Tensor q_start, int width, Tensor? reverse=None) -> Tensor")


def test_narrowpeak_suffix_mapping():
    from bionumpy_b200.io.delimited import NarrowPeakBuffer
    from bionumpy_b200.io.files import _buffer_type_for, _read_buffer_type_for, _suffix, bnp_open
    assert _suffix("peaks.narrowPeak.gz") == (".narrowPeak", True)
    assert _read_buffer_type_for(".narrowPeak") is NarrowPeakBuffer
    assert _buffer_type_for(".narrowPeak") is NarrowPeakBuffer
    with pytest.raises(NotImplementedError):
        bnp_open(os.path.join("/nonexistent", "x.narrowPeak"), "w")
    with pytest.raises(NotImplementedError):
        NarrowPeakBuffer.from_data(None)


def test_new_kernels_are_sm90a_code_without_stack_or_spills():
    tool = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(tool):
        pytest.skip("cuobjdump not available")
    out = subprocess.run([tool, "-res-usage", nv.LIB_PATH], capture_output=True, text=True).stdout
    usage = {m.group(1): (int(m.group(2)), int(m.group(3)))
             for m in re.finditer(r"Function (\S+):\s*REG:(\d+) STACK:(\d+)", out)}
    for name in KERNELS:
        found = [(n, v) for n, v in usage.items() if name in n]
        assert len(found) == 2, (name, found)          # the int64 and the float64 instance
        for _, (regs, stack) in found:
            assert stack == 0 and regs <= 64, (name, regs, stack)
    sass = subprocess.run([tool, "-sass", nv.LIB_PATH], capture_output=True, text=True).stdout
    assert "arch = sm_90a" in sass
    for block in re.split(r"\n\s+Function : ", sass):
        if any(n in block.split("\n", 1)[0] for n in KERNELS):
            assert "STL" not in block and "LDL" not in block          # no local-memory spills
