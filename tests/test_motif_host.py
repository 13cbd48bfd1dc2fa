"""Motif scores without a GPU: the oracle against the reference's goldens, the motif file readers, the argument checks
of the two C entry points, the missing-GPU error and the compiled code of the motif kernels."""
import ctypes
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch

import bionumpy_b200 as bnp
from bionumpy_b200 import _native as nv
from bionumpy_b200.sequence.position_weight_matrix import PWM, _pwm_from_counts

import motif_oracle as mo

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
DOC_DICT = {"A": [5, 1], "C": [1, 5], "G": [0, 0], "T": [0, 0]}
TEST_MATRIX = np.log([[0.4, 0.25], [0.1, 0.25], [0.4, 0.25], [0.1, 0.25]])


def _codes(text, alphabet="ACGT"):
    return mo.encode([text.encode()], alphabet)[0]


def test_oracle_docstring_golden():
    """position_weight_matrix.py:183-189, re-derived with NumPy."""
    matrix, alphabet = mo.from_dict(DOC_DICT)
    rows = ["ACTGAC", "CA", "GG"]
    flat, lens = mo.motif_scores(_codes("".join(rows)), [len(r) for r in rows], matrix)
    assert lens.tolist() == [5, 1, 1]
    assert flat.tolist() == [5.991464547107982, -np.inf, -np.inf, -np.inf, 5.991464547107982, 2.772588722239781,
                             -np.inf]
    assert mo.row_max(flat, lens).tolist() == [5.991464547107982, 2.772588722239781, -np.inf]


def test_oracle_reference_test_goldens():
    """tests/test_position_weight_matrix.py of the reference: test_window/test_pwm, test_sequence, test_sanity_motifs,
    test_a_motifs."""
    assert np.isclose(np.exp(mo.calculate_scores([0, 1], TEST_MATRIX)[0]), 0.1)
    assert np.allclose(np.exp(mo.calculate_scores([0, 1, 2, 3], TEST_MATRIX)[:3]), [0.1, 0.025, 0.1])
    neutral, _ = mo.from_dict({c: [0.25, 0.25] for c in "ACGT"})
    assert np.all(mo.calculate_scores([0, 1, 2, 3], neutral) == 0)
    a_matrix, _ = mo.from_dict({"A": [1, 1], "C": [0, 0], "G": [0, 0], "T": [0, 0]})
    assert mo.calculate_scores(_codes("AAC"), a_matrix).tolist() == [np.log(4 ** 2), -np.inf, -np.inf]


def test_package_matrix_bits_equal_the_oracle():
    for d in (DOC_DICT, {"A": [1, 1], "C": [0, 0], "G": [0, 0], "T": [0, 0]}, {c: [0.25, 0.25] for c in "ACGT"}):
        want, alphabet = mo.from_dict(d)
        pwm = PWM.from_dict(d)
        assert pwm.alphabet == alphabet and pwm.window_size == want.shape[1]
        assert np.array_equal(pwm._matrix.view(np.int64), want.view(np.int64))
    bg = {"A": 0.3, "C": 0.2, "G": 0.2, "T": 0.3}
    assert np.array_equal(PWM.from_dict(DOC_DICT, bg)._matrix, mo.from_dict(DOC_DICT, bg)[0])


def test_from_counts():
    counts = {"A": [3, 0, 10], "C": [1, 2, 0], "G": [0, 7, 0], "T": [6, 1, 0]}
    want, alphabet = mo.from_counts(counts)
    pwm = PWM.from_counts(counts)
    assert pwm.alphabet == alphabet == "ACGT"
    assert np.array_equal(pwm._matrix.view(np.int64), want.view(np.int64))
    assert np.allclose(np.exp(want).sum(axis=0), 1.0)
    assert np.array_equal(_pwm_from_counts(np.array(list(counts.values()))), want)


def test_read_motif_files():
    """test_read_csv_motif: str of pwm.csv equals str of pwm.jaspar (alphabet "ACE"); MA0080.1 keeps the JASPAR counts
    as log(count) - log(1/4), bit for bit."""
    csv, jaspar = bnp.io.read_motif(os.path.join(GOLDEN, "pwm.csv")), bnp.io.read_motif(os.path.join(GOLDEN, "pwm.jaspar"))
    assert str(csv) == str(jaspar)
    assert csv.alphabet == jaspar.alphabet == "ACE"
    assert str(csv) == mo.pwm_str(*mo.read_csv(os.path.join(GOLDEN, "pwm.csv")))
    ma = bnp.io.read_motif(os.path.join(GOLDEN, "MA0080.1.jaspar"))
    want, alphabet = mo.read_jaspar(os.path.join(GOLDEN, "MA0080.1.jaspar"))
    assert ma.alphabet == alphabet == "ACGT" and ma.window_size == 6
    assert np.array_equal(ma._matrix.view(np.int64), want.view(np.int64))
    assert ma._matrix[0, 0] == np.log(14.0) - np.log(0.25)
    assert ma._matrix[1, 2] == -np.inf


def _scores_call(lib, motif_len=6, alphabet_size=4, enc_mode=nv.ENC_ASCII_ACGT, lut=None, tail=0, matrix=1):
    z = ctypes.c_void_p(0)
    return lib.bnpk_rows_pwm_scores(z, 0, z, z, 0, enc_mode, lut, alphabet_size, ctypes.c_void_p(matrix), motif_len,
                                    tail, z, z, z, z)


def _max_call(lib, motif_len=6, alphabet_size=4, enc_mode=nv.ENC_ASCII_ACGT, lut=None, matrix=1):
    z = ctypes.c_void_p(0)
    return lib.bnpk_rows_pwm_max(z, 0, z, z, 0, enc_mode, lut, alphabet_size, ctypes.c_void_p(matrix), motif_len,
                                 z, z, z)


@pytest.mark.parametrize("call", [_scores_call, _max_call])
def test_entry_point_argument_errors(call):
    """No rows: a valid call returns 0 without touching the device; every bad argument is BNPK_E_BADARG."""
    lib = nv.load_library()
    lut = ctypes.c_void_p(1)
    assert call(lib) == 0
    assert call(lib, motif_len=1) == 0 and call(lib, motif_len=1024) == 0
    assert call(lib, alphabet_size=8, motif_len=1024, enc_mode=nv.ENC_LUT, lut=lut) == 0
    for kwargs in (dict(motif_len=0), dict(motif_len=1025), dict(motif_len=-1),
                   dict(alphabet_size=9, motif_len=1000, enc_mode=nv.ENC_LUT, lut=lut),
                   dict(alphabet_size=5, enc_mode=nv.ENC_ASCII_ACGT), dict(alphabet_size=3, enc_mode=nv.ENC_ASCII_ACTG),
                   dict(alphabet_size=1, enc_mode=nv.ENC_CODES), dict(alphabet_size=256, enc_mode=nv.ENC_CODES),
                   dict(enc_mode=4), dict(enc_mode=-1), dict(enc_mode=nv.ENC_LUT, lut=None),
                   dict(alphabet_size=5, enc_mode=nv.ENC_LUT, lut=None), dict(matrix=0)):
        assert call(lib, **kwargs) == nv.E_BADARG, kwargs
    if call is _scores_call:
        assert call(lib, tail=1) == 0 and call(lib, tail=2) == nv.E_BADARG


def test_python_limits_raise_before_any_launch():
    with pytest.raises(ValueError):
        bnp.get_motif_scores(["ACGT"], PWM(np.zeros((4, 1025)), "ACGT"))
    with pytest.raises(ValueError):
        bnp.get_motif_scores(["ACGT"], PWM(np.zeros((20, 500)), "ACDEFGHIKLMNPQRSTVWY"))


def test_get_motif_scores_needs_a_gpu():
    if torch.cuda.is_available():
        pytest.skip("has a GPU")
    pwm = PWM.from_dict(DOC_DICT)
    with pytest.raises(nv.NativeLibraryError):
        bnp.get_motif_scores(["ACTGAC", "CA"], pwm)
    with pytest.raises(nv.NativeLibraryError):
        pwm.calculate_scores("AAC")
    with pytest.raises(nv.NativeLibraryError):
        bnp.sequence.get_motif_scores("ACGTAC", pwm)


def _res_usage():
    tool = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(tool):
        pytest.skip("cuobjdump not available")
    out = subprocess.run([tool, "-res-usage", nv.LIB_PATH], capture_output=True, text=True).stdout
    return {m.group(1): (int(m.group(2)), int(m.group(3)))
            for m in re.finditer(r"Function (\S+):\s*REG:(\d+) STACK:(\d+)", out)}


def test_motif_kernels_are_sm90a_code_without_stack():
    usage = _res_usage()
    pwm = {n: v for n, v in usage.items() if re.search(r"rows_pwm_kernel|rows_pwm_generic_kernel", n)}
    assert len(pwm) == 10, sorted(pwm)                  # 2 modes x 4 encodings + 2 generic builds
    for name, (regs, stack) in pwm.items():
        assert stack == 0 and regs <= 64, (name, regs, stack)
    assert "sm_90a" in subprocess.run([shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump", "-res-usage", nv.LIB_PATH],
                                      capture_output=True, text=True).stdout


def test_existing_row_kernels_keep_their_registers():
    usage = _res_usage()
    # "<symbol> <registers>/<stack>" of every rows_kernel instantiation before the motif modes were added
    with open(os.path.join(GOLDEN, "rows_kernel_res_usage.txt")) as f:
        before = dict(line.split() for line in f if line.strip())
    rows = {n: v for n, v in usage.items() if "rows_kernel" in n}
    assert set(rows) == set(before)
    for name, (regs, stack) in rows.items():
        assert f"{regs}/{stack}" == before[name], name


def test_torch_library_registers_the_motif_op():
    from bionumpy_b200 import torch_ops
    assert hasattr(torch_ops.load(), "rows_pwm_scores")
    assert "bool tail" in str(torch._C._get_schema("bnpk::rows_pwm_scores", ""))
