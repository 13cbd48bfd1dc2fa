"""Intervals without a GPU: the NumPy interval oracle against the reference's goldens, the argument checks of the three
C entry points and the compiled code of the interval kernels."""
import ctypes
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

from bionumpy_b200 import _native as nv

import interval_oracle as io_

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
# tests/buffers.py:41-45 of the reference
BED6_TEXT = b"chr1\t1\t3\t.\t0\t-\nchr1\t40\t60\t.\t1\t+\nchr20\t400\t600\t.\t2\t+\n"
VALID_BED = b"chr1\t10\t20\nchr2\t20\t30\nchr1\t10\t20\nchr2\t20\t30\n"
MALFORMED_BED = b"chr1\t10\t20\nchr2\t10\ttwenty\n"


def test_bed6_buffer_golden():
    """tests/buffers.py 'bed' -> its three Bed6.single_entry records."""
    size, (chrom, start, stop, name, score, strand) = io_.parse_delimited(BED6_TEXT, io_.BED6)
    assert size == len(BED6_TEXT)
    assert chrom == [b"chr1", b"chr1", b"chr20"] and name == [b"."] * 3
    assert start.tolist() == [1, 40, 400] and stop.tolist() == [3, 60, 600] and score.tolist() == [0, 1, 2]
    assert strand.tolist() == [1, 0, 0]


def test_malformed_bed_line_numbers():
    """test_io_exceptions.py: line 1 in one buffer, line 4 * 100 + 1 through the reader at min_chunk_size = 200."""
    with pytest.raises(io_.Fault) as e:
        io_.parse_delimited(MALFORMED_BED, io_.BED)
    assert e.value.line == 1
    with pytest.raises(io_.Fault) as e:
        io_.read_delimited(VALID_BED * 100 + MALFORMED_BED, io_.BED, 200)
    assert e.value.line == 401


def test_carriage_return_bed():
    """test_io.py::test_carriage_return_bed: stop [2, 4]."""
    _, (chrom, start, stop) = io_.parse_delimited(b"chr1\t1\t2\r\nchr2\t3\t4\n", io_.BED)
    assert chrom == [b"chr1", b"chr2"] and start.tolist() == [1, 3] and stop.tolist() == [2, 4]


def test_delimited_buffers_intervals():
    """test_delimited_buffers.py: Interval(["chr1", "chr1"], [2, 10], [100, 20]) is this BED text."""
    _, (chrom, start, stop) = io_.parse_delimited(b"chr1\t2\t100\nchr1\t10\t20\n", io_.BED)
    assert chrom == [b"chr1"] * 2 and start.tolist() == [2, 10] and stop.tolist() == [100, 20]


def test_ten_column_file_read_as_intervals():
    import gzip
    data = gzip.open(os.path.join(GOLDEN, "ctcf.bed.gz")).read()
    chrom, start, stop = io_.read_delimited(data, io_.BED, 1 << 20)
    assert len(chrom) == 44722 == data.count(b"\n")
    first = data.split(b"\n", 1)[0].split(b"\t")
    assert (chrom[0], int(start[0]), int(stop[0])) == (first[0], int(first[1]), int(first[2]))


def _small_genome():
    raw = open(os.path.join(GOLDEN, "small_genome.fa"), "rb").read()
    index = io_.read_fai(open(os.path.join(GOLDEN, "small_genome.fa.fai")).read())
    return raw, index


def test_get_sequences_golden():
    """test_indexed_fasta.py::test_get_sequences: lengths [10, 39, 5, 100, 170], each the contig's slice."""
    raw, index = _small_genome()
    tuples = [("1", 10, 20), ("2", 11, 50), ("1", 5, 10), ("3", 10, 110), ("1", 80, 250)]
    flat, lens = io_.interval_sequences(raw, index, *zip(*tuples))
    assert lens.tolist() == [10, 39, 5, 100, 170]
    contigs = {}
    for block in raw.decode().split(">")[1:]:
        head, *lines = block.split("\n")
        contigs[head.split()[0]] = "".join(lines)
    offs = np.concatenate([[0], np.cumsum(lens)])
    for (c, a, b), o0, o1 in zip(tuples, offs[:-1], offs[1:]):
        assert bytes(flat[o0:o1]).decode() == contigs[c][a:b]


def test_strand_specific_sequences_golden():
    """test_dna.py::test_strand_specific_sequences: ['CG', 'CGT'] in DNAEncoding."""
    codes = np.array(["ACGT".index(c) for c in "ACGTACGTACGT"], dtype=np.uint8)
    rows = io_.strand_specific_sequences(codes, [1, 4], [3, 7], ["+", "-"], alphabet="ACGT")
    assert ["".join("ACGT"[c] for c in r) for r in rows] == ["CG", "CGT"]
    text = np.frombuffer(b"ACgTNx", dtype=np.uint8)
    assert bytes(io_.strand_specific_sequences(text, [0], [6], ["-"])[0]) == b"\0NA\0GT"


def _lib():
    return nv.load_library()


def test_delimited_columns_bad_arguments():
    lib = _lib()
    buf = ctypes.create_string_buffer(64)
    p = ctypes.cast(buf, ctypes.c_void_p)

    def call(kinds, outs=None, lens=None, n_columns=None, n_lines=1, status=p, columns=True):
        arr = (nv.Column * max(len(kinds), 1))()
        for i, k in enumerate(kinds):
            arr[i] = nv.Column(k, p.value if outs is None else outs[i], p.value if lens is None else lens[i])
        return lib.bnpk_delimited_columns(p, 64, p, p, n_lines, ctypes.cast(arr, ctypes.c_void_p) if columns else None,
                                          len(kinds) if n_columns is None else n_columns, status, None)

    assert call([nv.COL_TEXT], n_columns=0) == nv.E_BADARG
    assert call([nv.COL_INT] * 17) == nv.E_BADARG
    assert call([nv.COL_TEXT], columns=False) == nv.E_BADARG
    assert call([7]) == nv.E_BADARG
    assert call([-1]) == nv.E_BADARG
    assert call([nv.COL_INT], outs=[None]) == nv.E_BADARG
    assert call([nv.COL_STRAND], outs=[None]) == nv.E_BADARG
    assert call([nv.COL_TEXT], lens=[None]) == nv.E_BADARG
    assert call([nv.COL_TEXT], status=None) == nv.E_BADARG
    assert b"status" in lib.bnpk_last_error()
    assert call([nv.COL_SKIP], outs=[None], lens=[None], n_lines=0) == 0


def test_name_lookup_and_gather_bad_arguments():
    lib = _lib()
    buf = ctypes.create_string_buffer(64)
    p = ctypes.cast(buf, ctypes.c_void_p)
    lookup = [p, 64, p, p, 1, p, p, 1, p, p, None]
    for i in (0, 2, 3, 6, 8, 9):                   # base, starts, lens, name_offsets, out_ids, status
        args = list(lookup)
        args[i] = None
        assert lib.bnpk_name_lookup(*args) == nv.E_BADARG, i
    args = list(lookup)
    args[5] = None                                  # names with a non-empty table
    assert lib.bnpk_name_lookup(*args) == nv.E_BADARG
    args[4] = 0
    assert lib.bnpk_name_lookup(*args) == 0        # no rows: nothing to do
    # file, file_bytes, n_rows, ids, offset, lenc, lenb, len, n_contigs, start, stop, strand, lut, row_lens, offsets,
    # out, status, stream
    check = [p, 64, 1, p, p, p, p, p, 1, p, p, None, None, p, None, None, p, None]
    for i in (4, 5, 6, 7):                          # a contig column missing while ids are given
        args = list(check)
        args[i] = None
        assert lib.bnpk_interval_gather(*args) == nv.E_BADARG, i
    for i in (0, 9, 10, 13, 16):                   # file, start, stop, and the check pass' row_lens and status
        args = list(check)
        args[i] = None
        assert lib.bnpk_interval_gather(*args) == nv.E_BADARG, i
    args = list(check)
    args[11] = p                                    # a strand flag without the complement table
    assert lib.bnpk_interval_gather(*args) == nv.E_BADARG
    args = list(check)
    args[15] = p                                    # the copy pass without out_offsets
    assert lib.bnpk_interval_gather(*args) == nv.E_BADARG
    args = list(check)
    args[2] = 0
    assert lib.bnpk_interval_gather(*args) == 0


def test_interval_kernels_are_sm90a_code_without_stack():
    tool = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(tool):
        pytest.skip("cuobjdump not available")
    out = subprocess.run([tool, "-res-usage", nv.LIB_PATH], capture_output=True, text=True).stdout
    usage = {m.group(1): (int(m.group(2)), int(m.group(3)))
             for m in re.finditer(r"Function (\S+):\s*REG:(\d+) STACK:(\d+)", out)}
    found = {n: v for n, v in usage.items()
             if re.search(r"delimited_columns_kernel|name_lookup_kernel|interval_check_kernel|interval_copy_kernel", n)}
    assert len(found) == 4, sorted(found)
    for name, (regs, stack) in found.items():
        assert stack == 0 and regs <= 64 and "rows_kernel" not in name, (name, regs, stack)
