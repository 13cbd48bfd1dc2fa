"""String and pattern matching without a GPU: the oracle against the reference's goldens, the pattern parser and its
expansion, every argument error of the two C entry points, the missing-GPU error and the compiled match kernels."""
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
from bionumpy_b200.sequence.string_matcher import (FixedLenRegexMatcher, RegexMatcher, StringMatcher, _Pattern, expand,
                                                   parse_pattern)

import match_oracle as mo

T, F = True, False
TUTORIAL = ["CGTTAATTAC", "TCCTCCGGAAT", "TTGTCCTACACT", "ACCTAGCATACCC", "ATGTAGCGTCGACT", "CGCACGCTCGTTCAG",
            "GTCCACGTTAGTCCTG", "GGGTTAAGTAGTTTAGT", "CACAATGTTTCCGCTATG", "CGCTTCCAGGTTTTTAACC"]


def _b(rows):
    return [r.encode() for r in rows]


def test_oracle_docstring_golden():
    assert mo.matches(_b(["ACGT", "TACTAC"]), "AC", literal=True) == [[T, F, F], [F, T, F, F, T]]


def test_oracle_reference_test_goldens():
    """tests/test_string_matcher.py of the reference."""
    assert mo.matches(_b(["V1-1", "V2-1", "V1-1*2"]), "V1-1", literal=True) == [[T], [F], [T, F, F]]
    want = [[re.match("[AG].[AT]", s[o:o + 3]) is not None for o in range(len(s) - 2)] for s in ["ACGT", "AATGAT"]]
    assert mo.matches(_b(["ACGT", "AATGAT"]), "[AG].[AT]", alphabet="ACGT") == want
    assert mo.matches(_b(["ACGTTCG", "AATGAAAC"]), "AA.{,1}[CT]", "same", alphabet="ACGT") == \
        [[F] * 7, [T, F, F, F, T, T, F, F]]
    assert mo.matches(_b(["ACA", "TACTAC"]), "AC", literal=True, alphabet="ACGT") == [[T, F], [F, T, F, F, T]]


def test_oracle_integration_and_tutorial_goldens():
    aa = "ACDEFGHIKLMNPQRSTVWY*"
    assert mo.matches(_b(["AAACCC", "EEAAF"]), "AA", "same", alphabet=aa) == [[T, T, F, F, F, F], [F, F, T, F, F]]
    assert mo.counts(_b(TUTORIAL), "AC", literal=True).tolist() == [1, 0, 2, 2, 1, 1, 1, 0, 1, 1]


def test_oracle_validates_encoded_rows():
    with pytest.raises(mo.OracleEncodingError) as e:
        mo.matches(_b(["ACGT", "acNt"]), "AC", alphabet="ACGT")
    assert e.value.offset == 6


@pytest.mark.parametrize("pattern, want", [
    ("AC", [[{"A"}, {"C"}]]),
    ("[AG].[AT]", [[{"A", "G"}, None, {"A", "T"}]]),
    ("AA.{,1}[CT]", [[{"A"}, {"A"}, {"C", "T"}], [{"A"}, {"A"}, None, {"C", "T"}]]),
    ("A.{1,2}C.{0,1}G", [[{"A"}, None, {"C"}, {"G"}], [{"A"}, None, {"C"}, None, {"G"}],
                          [{"A"}, None, None, {"C"}, {"G"}], [{"A"}, None, None, {"C"}, None, {"G"}]]),
    ("...", [[None, None, None]]),
    ("[.]", [[{"."}]]),
])
def test_parser_expansion(pattern, want):
    assert expand(parse_pattern(pattern)) == want


@pytest.mark.parametrize("pattern", ["", "A*", "A+", "A?", "A|C", "(AC)", "A.{3}C", "A[]C", "[AC", "AC]", ".{1,2}A",
                                     "A.{1,2}", "A.{3,1}C", "A.{1,2}.{1,2}C", "A{2}", "^A", "A$", "A\\C", "[^A]", "[A-C]"])
def test_parser_rejects_what_is_outside_the_grammar(pattern):
    with pytest.raises(ValueError):
        expand(parse_pattern(pattern))


def test_literal_patterns_take_every_character():
    assert expand(parse_pattern("A.*[", literal=True)) == [[{"A"}, {"."}, {"*"}, {"["}]]


def test_pattern_limits_and_encoding_errors_before_any_launch():
    with pytest.raises(ValueError):
        StringMatcher("A" * 1025, bnp.DNAEncoding)
    with pytest.raises(ValueError):
        RegexMatcher("A.{0,64}C", bnp.DNAEncoding)                      # 65 sub-patterns
    with pytest.raises(ValueError):
        RegexMatcher("A.{0,5}C.{0,10}G", bnp.DNAEncoding)               # 66 sub-patterns
    with pytest.raises(ValueError):
        FixedLenRegexMatcher("A" * 1025, bnp.encodings.BaseEncoding)
    with pytest.raises(ValueError):                                     # 8 words per raw-byte column: 1025 columns
        RegexMatcher("A" * 500 + ".{0,1}" + "C" * 24, bnp.encodings.BaseEncoding)
    with pytest.raises(ValueError):
        FixedLenRegexMatcher("A.{1,2}C", bnp.DNAEncoding)
    with pytest.raises(bnp.EncodingError) as e:
        StringMatcher("ACN", bnp.DNAEncoding)
    assert e.value.offset == 2
    with pytest.raises(bnp.EncodingError):
        FixedLenRegexMatcher("[AU]C", bnp.DNAEncoding)
    with pytest.raises(TypeError):
        bnp.match_string(bnp.EncodedArray(torch.zeros(3, dtype=torch.uint8), bnp.KmerEncoding(bnp.DNAEncoding, 2)), "A")


def test_pattern_sets_and_lengths():
    p = _Pattern("A.{0,1}[ct]", bnp.DNAEncoding)
    assert p.sub_lens == [2, 3] and p.span == 3 and p.alphabet_size == 4
    assert p._words.tolist() == [1, 0b1010, 1, 0b1111, 0b1010]
    raw = _Pattern("a.", bnp.encodings.BaseEncoding, literal=True)
    assert raw.alphabet_size == 256 and raw._words.reshape(2, 8)[0].tolist() == [0, 0, 0, 1 << 1, 0, 0, 0, 0]
    assert raw._words.reshape(2, 8)[1, 1] == 1 << (ord(".") - 32)
    dot = _Pattern("a.", bnp.encodings.BaseEncoding)
    assert (dot._words.reshape(2, 8)[1] == -1).all()


def _call(lib, count, alphabet_size=4, enc_mode=nv.ENC_ASCII_ACGT, lut=None, sets=1, sub_lens=(3,), n_sub=None,
          same=0):
    z = ctypes.c_void_p(0)
    lens = (ctypes.c_int32 * max(len(sub_lens), 1))(*sub_lens)
    n = len(sub_lens) if n_sub is None else n_sub
    args = [z, 0, z, z, 0, enc_mode, lut, alphabet_size, ctypes.c_void_p(sets), ctypes.cast(lens, ctypes.c_void_p), n,
            same]
    if count:
        return lib.bnpk_rows_match_count(*args, z, z, z)
    return lib.bnpk_rows_match(*args, z, z, z, z)


@pytest.mark.parametrize("count", [False, True])
def test_entry_point_argument_errors(count):
    """No rows: a valid call returns 0 without touching the device; every bad argument is BNPK_E_BADARG."""
    lib = nv.load_library()
    lut = ctypes.c_void_p(1)
    assert _call(lib, count) == 0
    assert _call(lib, count, same=1) == 0
    assert _call(lib, count, sub_lens=(1,)) == 0 and _call(lib, count, sub_lens=(1024,)) == 0
    assert _call(lib, count, sub_lens=tuple(range(1, 65))) == 0 and _call(lib, count, sub_lens=(1024,) * 8) == 0
    assert _call(lib, count, alphabet_size=256, enc_mode=nv.ENC_CODES, sub_lens=(1024,)) == 0
    assert _call(lib, count, alphabet_size=21, enc_mode=nv.ENC_LUT, lut=lut) == 0
    for kwargs in (dict(sub_lens=(0,)), dict(sub_lens=(1025,)), dict(sub_lens=(-1,)), dict(sub_lens=(3, 0)),
                   dict(sub_lens=(1,) * 65), dict(sub_lens=(3,), n_sub=0), dict(sub_lens=(1024,) * 8 + (1,)),
                   dict(alphabet_size=256, enc_mode=nv.ENC_CODES, sub_lens=(1024, 1)),
                   dict(alphabet_size=256, enc_mode=nv.ENC_LUT, lut=lut), dict(alphabet_size=257, enc_mode=nv.ENC_CODES),
                   dict(alphabet_size=1, enc_mode=nv.ENC_CODES), dict(alphabet_size=5, enc_mode=nv.ENC_ASCII_ACGT),
                   dict(alphabet_size=3, enc_mode=nv.ENC_ASCII_ACTG), dict(enc_mode=4), dict(enc_mode=-1),
                   dict(enc_mode=nv.ENC_LUT, lut=None), dict(sets=0), dict(same=2), dict(same=-1)):
        assert _call(lib, count, **kwargs) == nv.E_BADARG, kwargs


def test_match_string_needs_a_gpu():
    if torch.cuda.is_available():
        pytest.skip("has a GPU")
    with pytest.raises(nv.NativeLibraryError):
        bnp.match_string(["ACGT", "TACTAC"], "AC")
    with pytest.raises(nv.NativeLibraryError):
        bnp.sequence.match_string("ACGTAC", "AC")
    with pytest.raises(nv.NativeLibraryError):
        RegexMatcher("AA.{,1}[CT]", bnp.DNAEncoding).rolling_window(["ACGTTCG"])


def _res_usage():
    tool = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(tool):
        pytest.skip("cuobjdump not available")
    out = subprocess.run([tool, "-res-usage", nv.LIB_PATH], capture_output=True, text=True).stdout
    return {m.group(1): (int(m.group(2)), int(m.group(3)))
            for m in re.finditer(r"Function (\S+):\s*REG:(\d+) STACK:(\d+)", out)}


def test_match_kernels_have_no_stack_frame():
    usage = _res_usage()
    match = {n: v for n, v in usage.items() if re.search(r"rows_match_kernel|rows_match_generic_kernel", n)}
    assert len(match) == 10, sorted(match)              # 2 modes x 4 encodings + 2 generic builds
    for name, (regs, stack) in match.items():
        assert stack == 0 and regs <= 128, (name, regs, stack)


def test_torch_library_registers_the_match_op():
    from bionumpy_b200 import torch_ops
    assert hasattr(torch_ops.load(), "rows_match")
    assert "int[] sub_lens" in str(torch._C._get_schema("bnpk::rows_match", ""))


def test_exports():
    assert bnp.match_string is bnp.sequence.match_string
    assert bnp.sequence.StringMatcher is StringMatcher and bnp.sequence.RegexMatcher is RegexMatcher
