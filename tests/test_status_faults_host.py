"""The fault word status[ST_BAD_BASE] is decoded in ops.py alone: every ScanStatus decoder on hand-built words, the
one-copy read-back on CPU tensors, no other module unpacking a fault, and (GPU) the device-to-host copies of every
path that reads a fault back."""
import gzip
import os
import re

import pytest
import torch

from bionumpy_b200 import _native as nv
from bionumpy_b200 import ops

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")


def _status(fault):
    words = [0] * nv.ST_WORDS
    words[nv.ST_BAD_BASE] = fault
    return ops.ScanStatus(words)


# the packers of csrc/bnpk_device.cuh, restated
def _row_pos(row, pos):
    return row << 32 | pos


def _column(line, column, kind):
    return line << 8 | column << 3 | kind


def _record(record, kind):
    return record << 8 | kind


def test_sentinel_is_no_fault_in_every_decoder():
    st = _status(nv.INT64_MAX)
    assert st.fault is None
    assert st.bad_base() is None and st.bad_base(10) is None
    assert st.bad_base_offset(torch.tensor([3, 4], dtype=torch.int32)) is None
    assert st.column_fault() is None and st.record_fault() is None


def test_plain_index():
    for v in (0, 1, 12345, nv.INT64_MAX - 1):
        assert _status(v).fault == v


def test_row_position():
    assert _status(_row_pos(0, 0)).bad_base() == (0, 0)
    assert _status(_row_pos(7, 3)).bad_base(8) == (7, 3)
    top = (1 << 31) - 1                        # the largest row and position: int32 row counts and lengths
    assert _status(_row_pos(top, top)).bad_base() == (top, top)


def test_row_past_n_rows_is_not_a_bad_base_of_these_rows():
    st = _status(_row_pos(5, 2))
    assert st.bad_base(5) is None and st.bad_base(6) == (5, 2) and st.bad_base() == (5, 2)
    assert st.bad_base_offset(torch.ones(5, dtype=torch.int32)) is None
    assert st.fault == _row_pos(5, 2)


def test_flat_offset():
    lens = torch.tensor([3, 0, 4, 2], dtype=torch.int32)
    assert _status(_row_pos(0, 2)).bad_base_offset(lens) == 2
    assert _status(_row_pos(2, 1)).bad_base_offset(lens) == 3 + 0 + 1
    assert _status(_row_pos(3, 1)).bad_base_offset(lens) == 3 + 0 + 4 + 1


def test_column_layout():
    for kind in (nv.BAD_TABS, nv.BAD_COLUMNS, nv.BAD_INT, nv.BAD_STRAND):
        assert _status(_column(0, 0, kind)).column_fault() == (0, 0, kind)
        assert _status(_column(17, 5, kind)).column_fault() == (17, 5, kind)
    top = (1 << 55) - 1                        # the largest line below the sentinel's bits
    assert _status(_column(top, 31, nv.BAD_STRAND)).column_fault() == (top, 31, nv.BAD_STRAND)


def test_record_layout():
    for kind in (nv.BAM_BAD_BLOCK_SIZE, nv.BAM_BAD_REF_ID, nv.BAM_BAD_NAME, nv.BAM_BAD_SIZES, nv.BAM_BAD_CIGAR_OP):
        assert _status(_record(0, kind)).record_fault() == (0, kind)
        assert _status(_record(123456, kind)).record_fault() == (123456, kind)
    top = (1 << 55) - 1
    assert _status(_record(top, nv.BAM_BAD_CIGAR_OP)).record_fault() == (top, nv.BAM_BAD_CIGAR_OP)


def test_read_back_order_and_one_copy(monkeypatch):
    calls = []
    cpu = torch.Tensor.cpu

    def counted(self, *a, **k):
        calls.append(self.numel())
        return cpu(self, *a, **k)

    monkeypatch.setattr(torch.Tensor, "cpu", counted)
    a = torch.arange(nv.ST_WORDS, dtype=torch.int64)
    b = torch.arange(nv.ST_WORDS + 1, dtype=torch.int64) + 100          # a longer block: its first ST_WORDS words
    b[nv.ST_BAD_BASE] = nv.INT64_MAX
    count = torch.tensor([7], dtype=torch.int32)
    total = torch.tensor(9, dtype=torch.int64)
    st_a, n, st_b, t = ops.read_back(a, count, b, total)
    assert calls == [2 * nv.ST_WORDS + 2]
    assert st_a.words == list(range(nv.ST_WORDS)) and st_a.fault == nv.ST_BAD_BASE
    assert st_b.words == [100 + i if i != nv.ST_BAD_BASE else nv.INT64_MAX for i in range(nv.ST_WORDS)]
    assert st_b.fault is None
    assert (n, t) == (7, 9) and type(n) is int
    assert ops.read_back() == [] and calls == [2 * nv.ST_WORDS + 2]


def test_only_ops_decodes_the_fault_word():
    """No module but ops.py and _native.py names ST_BAD_BASE, compares with INT64_MAX or shifts a fault by 8."""
    pattern = re.compile(r"ST_BAD_BASE|INT64_MAX|>> 8\b|<< 8 \|")
    pkg = os.path.join(ROOT, "bionumpy_b200")
    found = []
    for d, _, files in os.walk(pkg):
        for f in files:
            path = os.path.join(d, f)
            if not f.endswith(".py") or os.path.relpath(path, pkg) in ("ops.py", "_native.py"):
                continue
            for i, line in enumerate(open(path), 1):
                code = line.split("#")[0]
                if pattern.search(code) and "INT64_MIN" not in code:
                    found.append(f"{os.path.relpath(path, ROOT)}:{i}: {line.strip()}")
    assert not found, found


def test_device_faults_are_reported_through_one_helper():
    """Outside bnpk_device.cuh only the warp-specialised count (tile_ws_kernel.inl) atomicMin-s into BAD_BASE."""
    csrc = os.path.join(ROOT, "bionumpy_b200", "csrc")
    found = []
    for f in sorted(os.listdir(csrc)):
        if f in ("bnpk_device.cuh", "tile_ws_kernel.inl"):
            continue
        text = open(os.path.join(csrc, f)).read()
        found += [f for line in text.splitlines() if "atomicMin" in line and "BNPK_ST_BAD_BASE" in line]
        found += [f for name in ("report_bad(", "col_fault(", " report(") if name in text]
    assert not found, found


# ---- device-to-host copies of each path that reads a fault back (GPU) ------------------------------------------------
# Each path makes exactly these copies (.cpu(), .item() and .tolist() of CUDA tensors) on its good path.
COPIES = {
    "get_pileup": 1, "merge_intervals": 1, "from_intervals": 1, "get_interval_sequences": 1, "bed_from_raw_buffer": 2,
    "delimited_text": 1, "formatted": 1, "bam_chunk": 1, "concatenate": 1,
}


def _paths():
    import bionumpy_b200 as bnp
    from bionumpy_b200.arithmetics import get_pileup, merge_intervals
    from bionumpy_b200.datatypes import concatenate
    from bionumpy_b200.genomic_data.genome import GenomicIntervals
    from bionumpy_b200.io import bam, write
    from bionumpy_b200.io.delimited import BedBuffer, Bed6Buffer, DelimitedText
    from bionumpy_b200.io.indexed_fasta import IndexedFasta

    bed = b"chr1\t3\t8\tr0\t0\t+\nchr1\t5\t7\tr1\t0\t-\nchr2\t10\t12\tr2\t0\t.\n"
    chunk = torch.frombuffer(bytearray(bed), dtype=torch.uint8).cuda()
    bed6 = Bed6Buffer.from_raw_buffer(chunk).get_data()
    iv = bnp.Interval(["chr1", "chr1", "chr2"], [3, 5, 10], [8, 7, 12])
    genome = bnp.Genome.from_dict({"chr1": 100, "chr2": 80})
    fa = IndexedFasta(os.path.join(GOLDEN, "small_genome.fa"))
    name = list(fa._index)[0]
    on_fa = bnp.Interval([name, name], torch.tensor([0, 2]).cuda(), torch.tensor([4, 6]).cuda())
    reads = bnp.SequenceEntry(["a", "b"], ["ACGT", "GGA"])
    data = gzip.open(os.path.join(GOLDEN, "alignments.bam")).read()
    header = bam.parse_header(data)
    records = torch.frombuffer(bytearray(data[header.size:]), dtype=torch.uint8).cuda()
    bam_buffer = bam.BamBuffer.modify_class_with_header_data(header)
    torch.cuda.synchronize()
    return {
        "get_pileup": lambda: get_pileup(iv, 100),
        "merge_intervals": lambda: merge_intervals(iv),
        "from_intervals": lambda: GenomicIntervals.from_intervals(iv, genome),
        "get_interval_sequences": lambda: fa.get_interval_sequences(on_fa),
        "bed_from_raw_buffer": lambda: BedBuffer.from_raw_buffer(chunk),
        "delimited_text": lambda: DelimitedText(bed6),
        "formatted": lambda: write.formatted_entries(reads, nv.FMT_FASTA),
        "bam_chunk": lambda: bam_buffer.read_device_chunk(records, True, 0),
        "concatenate": lambda: concatenate(bed6, bed6),
    }


@pytest.mark.gpu
def test_each_path_keeps_its_copies(monkeypatch):
    paths = _paths()
    copies = []
    for method in ("cpu", "item", "tolist"):
        original = getattr(torch.Tensor, method)

        def counted(self, *a, _original=original, **k):
            if self.is_cuda:
                copies.append(1)
            return _original(self, *a, **k)

        monkeypatch.setattr(torch.Tensor, method, counted)
    got = {}
    for name, fn in paths.items():
        fn()                                   # warm: name tables and device LUTs are built once
        copies.clear()
        fn()
        got[name] = len(copies)
    assert got == COPIES
