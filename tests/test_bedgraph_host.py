"""bedGraph and float tracks without a GPU: tests/bedgraph_oracle.py pinned to the reference guide's per-peak maxima and
means on the fixtures, the decimal grammar, the host-built power-of-five table against an independent exact
computation, the C-ABI constants and dispatcher schemas, and the machine code of the new kernels."""
import io
import math
import os
import re
import shutil
import subprocess
from fractions import Fraction

import numpy as np
import pytest

import bedgraph_oracle as oracle
from bionumpy_b200 import _native as nv
from bionumpy_b200.io.decimal import pow5_words
from bionumpy_b200.io.delimited import BdgBuffer, BedGraphBuffer

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
GUIDE_MAX = [227, 231, 412, 296, 165, 163, 271, 148, 268, 568, 1901, 90, 236]
GUIDE_MEAN = [145.68181818, 147.86129032, 256.671875, 187.71202532, 106.79934211, 106.23355263, 173.04501608,
              96.27152318, 169.59235669, 346.37272727, 593.44084507, 60.25614035, 150.72580645]
KERNELS = ("parse_float_kernel", "track_f64_locate_kernel", "track_f64_scan_kernel", "track_f64_reduce_kernel",
           "track_f64_fold_kernel", "track_f64_combine_kernel")
REG_CAP = {"parse_float_kernel": 48, "track_f64_combine_kernel": 96}         # every other new kernel: 64


def test_oracle_reproduces_the_guide():
    sizes = oracle.read_sizes(os.path.join(GOLDEN, "small.chrom.sizes"))
    dense = oracle.dense_track(oracle.read_bedgraph(os.path.join(GOLDEN, "small_treat_pileup.bdg")), sizes)
    peaks = oracle.read_bed(os.path.join(GOLDEN, "small_peaks.narrowPeak"))
    mx = oracle.interval_max(dense, peaks)
    assert mx == GUIDE_MAX
    assert np.allclose(oracle.interval_mean(dense, peaks), GUIDE_MEAN, rtol=0, atol=5e-9)
    assert sum(m > 200 for m in mx) == 9
    # math.fsum agrees with the exact sum on these values
    c, s, e = peaks[0]
    assert math.fsum(dense[c][s:e]) == float(oracle.exact_sum(dense[c][s:e]))


def test_oracle_reads_the_small_fixture():
    rows = oracle.read_bedgraph(os.path.join(GOLDEN, "small.bdg"))
    assert rows[0] == ("chr1", 0, 9800, -0.0) and math.copysign(1, rows[0][3]) == -1
    assert len(rows) == 99


def test_oracle_gap_fill_and_overlap_rule():
    d = oracle.dense_track([("a", 2, 4, 1.5), ("a", 6, 7, -0.0)], {"a": 8})
    assert d["a"].tolist() == [0, 0, 1.5, 1.5, 0, 0, -0.0, 0]
    with pytest.raises(ValueError):
        oracle.dense_track([("a", 2, 4, 1.5), ("a", 3, 7, 1.0)], {"a": 8})
    with pytest.raises(ValueError):
        oracle.dense_track([("a", 2, 9, 1.5)], {"a": 8})
    with pytest.raises(KeyError):
        oracle.dense_track([("b", 2, 3, 1.5)], {"a": 8})


@pytest.mark.parametrize("text", ["0", "-0", "+.5", "5.", "1e5", "1E-5", "0.000", "1" + "0" * 30,
                                  "0.00000000001234567890123456789", "1234567890123456789", "00012e+0003"])
def test_grammar_accepts(text):
    assert oracle.parse(text) == float(text)


@pytest.mark.parametrize("text", ["", ".", "-", "e1", "1e", "1.2.3", "nan", "inf", "0x10", "1_0", " 1", "1 ",
                                  "12345678901234567891", "1.0000000000000000001"])
def test_grammar_rejects(text):
    with pytest.raises(ValueError):
        oracle.parse(text)


def test_pow5_table_against_an_exact_computation():
    """Every entry is 5^q scaled into [2^127, 2^128): truncated for q >= 0, and for q < 0 no more than one above the
    truncation of the exact value (it is a rounded-up reciprocal); q = 0 and q = -1 are the published words."""
    words = pow5_words()
    assert words.dtype == np.uint64 and words.size == 2 * (nv.POW5_MAX - nv.POW5_MIN + 1)
    for i, q in enumerate(range(nv.POW5_MIN, nv.POW5_MAX + 1)):
        entry = int(words[2 * i]) << 64 | int(words[2 * i + 1])
        x = Fraction(5) ** q
        k = 127 - (x.numerator.bit_length() - x.denominator.bit_length())
        scaled = x * Fraction(2) ** k
        while scaled >= 2 ** 128:
            scaled /= 2
        while scaled < 2 ** 127:
            scaled *= 2
        floor = scaled.numerator // scaled.denominator
        assert 2 ** 127 <= entry < 2 ** 128, q
        if q >= 0:
            assert entry == floor, q
        else:
            assert floor <= entry <= floor + 1, q
    i0 = -nv.POW5_MIN
    assert (int(words[2 * i0]), int(words[2 * i0 + 1])) == (0x8000000000000000, 0)
    assert (int(words[2 * i0 - 2]), int(words[2 * i0 - 1])) == (0xCCCCCCCCCCCCCCCC, 0xCCCCCCCCCCCCCCCD)


def test_header_constants():
    text = open(os.path.join(ROOT, "include", "bnpk.h")).read()
    for name, val in (("BNPK_BAD_FLOAT", nv.BAD_FLOAT), ("BNPK_OP_DIV", nv.OP_DIV), ("BNPK_BAD_CIGAR", nv.BAD_CIGAR)):
        m = re.search(rf"#define\s+{name}\s+(\d+)", text)
        assert m and int(m.group(1)) == val, name
    assert nv.BAD_FLOAT == 7          # the last kind the 3-bit field of a column fault holds
    assert "#define BNPK_ABI_VERSION 3" in text


def test_read_header_skips_track_browser_and_comment_lines():
    f = io.BytesIO(b"track type=bedGraph\nbrowser position chr1:1-10\n#x\nchr1\t0\t1\t0.5\n")
    assert BedGraphBuffer.read_header(f) == "track type=bedGraph\nbrowser position chr1:1-10\n#x\n"
    assert f.read() == b"chr1\t0\t1\t0.5\n"
    assert issubclass(BedGraphBuffer, BdgBuffer)


def test_bdg_opens_for_reading_with_bedgraph_buffer():
    from bionumpy_b200.io.files import _buffer_type_for, _read_buffer_type_for
    assert _read_buffer_type_for(".bdg") is BedGraphBuffer
    assert _buffer_type_for(".bdg") is BdgBuffer
    with pytest.raises(NotImplementedError):
        BdgBuffer.from_raw_buffer(b"x\t0\t1\t0.5\n")


def test_dispatcher_schemas():
    import torch
    lib = os.path.join(os.path.dirname(nv.LIB_PATH), "libbnpk_torch.so")
    if not os.path.exists(lib):
        pytest.skip("libbnpk_torch.so not built")
    torch.ops.load_library(lib)
    want = {
        "parse_float": "bnpk::parse_float(Tensor base, Tensor starts, Tensor lens, int column, Tensor pow5_table) -> "
                       "(Tensor, Tensor)",
        "track_f64_reduce": "bnpk::track_f64_reduce(Tensor run_starts, Tensor values, Tensor q_start, Tensor q_stop, "
                            "int mode) -> Tensor",
        "track_f64_combine": "bnpk::track_f64_combine(Tensor a_starts, Tensor a_values, Tensor b_starts, "
                             "Tensor b_values, int op) -> (Tensor, Tensor, Tensor)",
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
    for name in KERNELS:
        found = [(n, v) for n, v in usage.items() if name in n]
        assert len(found) == 1, (name, found)
        regs, stack = found[0][1]
        assert stack == 0 and regs <= REG_CAP.get(name, 64), (name, regs, stack)
    sass = subprocess.run([tool, "-sass", nv.LIB_PATH], capture_output=True, text=True).stdout
    assert "arch = sm_90a" in sass
    for block in re.split(r"\n\s+Function : ", sass):
        if any(n in block.split("\n", 1)[0] for n in KERNELS):
            assert "STL" not in block and "LDL" not in block          # no local-memory spills
