"""The ctypes ops (bionumpy_b200.ops) check every tensor they hand to libbnpk.so before they allocate or launch
anything, with the dispatcher's rules: contiguous CUDA tensors of the stated dtype, LUTs of 256 uint8, offsets of at
least R + 1 int64, a hist of at least n_bins int64, a status block of ST_WORDS int64 words, an ``out`` that holds what
the call writes, one length per start.  Every rejection runs against a library that fails the test when it is called,
so a missing check is a test failure and never a bad pointer in a kernel; bnpk_launch_count() stays put."""
import numpy as np
import pytest
import torch

from bionumpy_b200 import _native as nv
from bionumpy_b200 import ops

pytestmark = pytest.mark.gpu
DEV = "cuda"
ROWS = [b"ACGTACGTTGCA", b"GGGCCCAATT", b"TTTTACGTAGCTAGCT"]
NAMES = [b"r0", b"r1", b"r2"]
FASTQ = b"@r\nACGTACGT\n+\nIIIIIIII\n@s\nTTGCAACG\n+\nIIIIIIII\n"
FASTA = b">a\nAC\nGT\n>b\nTT\n>c\n"
BED = b"chr1\t5\t+\nchr2\t7\t-\n"
BINS = 1024


def _u8(data, device=DEV):
    return torch.from_numpy(np.frombuffer(data, dtype=np.uint8).copy()).to(device)


def _t(values, dtype=torch.int64):
    return torch.tensor(values, dtype=dtype, device=DEV)


def _view(rows):
    """(base uint8, starts int64, lens int32) of the rows laid end to end on the device."""
    lens = [len(r) for r in rows]
    return _u8(b"".join(rows)), _t(np.cumsum([0] + lens[:-1]).tolist()), _t(lens, torch.int32)


def _valid(op):
    """Valid arguments of every op, by name; the lines of the FASTA and BED chunks come from ops.line_split."""
    a = dict(zip(("base", "starts", "lens"), _view(ROWS)))
    a["lut"] = torch.full((256,), 255, dtype=torch.uint8, device=DEV)
    a["lut"][torch.tensor(list(b"ACGT"))] = _t(range(4), torch.uint8)
    a["offsets"] = _t(np.cumsum([0] + [len(r) for r in ROWS]).tolist())
    a["total"] = int(a["offsets"][-1])
    a.update(status=nv.new_status(DEV), hist=torch.zeros(BINS, dtype=torch.int64, device=DEV),
             out=torch.empty(a["total"], dtype=torch.uint8, device=DEV), chunk=_u8(FASTQ),
             chunk_host=_u8(FASTQ, "cpu"), lut_host=a["lut"].cpu(), synth_out=_u8(bytes(2 * 317)))
    a.update(keys=_t([-1] * BINS), counts=_t([0] * BINS), n_used=_t([0]), new_keys=_t([-1] * 2 * BINS),
             new_counts=_t([0] * 2 * BINS), matrix=torch.ones(3, 4, dtype=torch.float64, device=DEV),
             sets=_t([1, 2], torch.int32), values=_t([0, 1, 2, 3]), row_bounds=_t([0, 2, 4]),
             hash_offsets=_t([5, 7]), mask=torch.zeros(64, dtype=torch.uint8, device=DEV))
    a.update(start=_t([0, 3]), stop=_t([5, 10]), same_prev=_t([0, 1], torch.uint8), strand=_t([0, 1], torch.uint8),
             iv_offsets=_t([0, 5, 12]), run_starts=_t([0, 5, 10]), run_values=_t([1, 2]), q_start=_t([0, 3]),
             out_offsets=_t([0, 2, 4]), contig_ends=_t([0, 4, 10]))
    a["fasta"] = _u8(FASTA)
    a["f_starts"], a["f_lens"], _ = ops.line_split(a["fasta"], 1, 0, 0, ord(">"), False, 0, max_rows=FASTA.count(b"\n"))
    is_header, _ = ops.multiline_flags(a["fasta"], a["f_starts"], a["f_lens"])
    # the lines of the complete entries a and b
    a["is_header"], a["f_starts"], a["f_lens"] = is_header[:5], a["f_starts"][:5], a["f_lens"][:5]
    a["hdr_before"] = ops.row_offsets(a["is_header"])
    a["bed"] = _u8(BED)
    a["b_starts"], a["b_lens"], _ = ops.line_split(a["bed"], 1, 0, 0, ord("#"), False, 0, max_rows=2)
    a.update(names=_view(NAMES), name_table=_u8(b"r0r1r2"), name_offsets=_t([0, 2, 4, 6]),
             strand_col=_t([0, 1, 2], torch.uint8), text_out=torch.empty(8, dtype=torch.uint8, device=DEV))
    a["rec_offsets"], _ = ops.format_offsets(nv.FMT_FASTA, 1, _fields(a))
    a["line_offsets"], _ = ops.delimited_offsets(_columns(a))
    keys, _, _, _ = ops.interval_events(a["start"], a["stop"], size=10)
    a["sorted_keys"] = torch.sort(keys).values
    if op == "HostPipeline.kmer_count":
        a["pipeline"] = ops.HostPipeline(1 << 16)
    return a


def _fields(a):
    return (a["names"] + (None,), (a["base"], a["starts"], a["lens"], a["lut"]), None)


def _columns(a):
    return [(nv.COL_TEXT, a["names"]), (nv.COL_INT, a["values"][:3]), (nv.COL_STRAND, a["strand_col"])]


def _rows(a):
    return a["base"], a["starts"], a["lens"]


# op -> (the arguments the rejections below change, the first being a device tensor; the call)
OPS = {
    "count_byte": ("chunk", lambda a: ops.count_byte(a["chunk"], 10)),
    "line_split": ("chunk", lambda a: ops.line_split(a["chunk"], 4, 1)),
    "chunk_kmer_count": ("chunk lut hist status", lambda a: ops.chunk_kmer_count(
        a["chunk"], 5, BINS, hist=a["hist"], enc_mode=nv.ENC_LUT, lut=a["lut"], status=a["status"])),
    "row_offsets": ("lens", lambda a: ops.row_offsets(a["lens"], 1)),
    "rows_encode": ("base starts lut offsets status", lambda a: ops.rows_encode(
        *_rows(a), nv.ENC_LUT, a["lut"], a["offsets"], a["status"], a["total"])),
    "rows_kmer_hash": ("base starts lut offsets status", lambda a: ops.rows_kmer_hash(
        *_rows(a), nv.ENC_LUT, 5, a["lut"], a["offsets"], a["status"], a["total"])),
    "rows_generic_hash": ("base starts lut offsets status", lambda a: ops.rows_generic_hash(
        *_rows(a), 5, 3, a["lut"], a["offsets"], a["status"], a["total"])),
    "rows_minimizers": ("base starts lut offsets status", lambda a: ops.rows_minimizers(
        *_rows(a), nv.ENC_LUT, 5, 7, a["lut"], a["offsets"], a["status"], a["total"])),
    "rows_kmer_count": ("base starts lut hist status", lambda a: ops.rows_kmer_count(
        *_rows(a), nv.ENC_LUT, 5, BINS, 0, a["lut"], a["hist"], status=a["status"])),
    "rows_reverse_complement": ("base starts lut offsets", lambda a: ops.rows_reverse_complement(
        *_rows(a), a["lut"], a["offsets"], a["total"])),
    "rows_kmer_hash_canonical": ("base starts lut offsets status", lambda a: ops.rows_kmer_hash_canonical(
        *_rows(a), nv.ENC_LUT, 5, 3, a["lut"], a["offsets"], a["status"], a["total"])),
    "rows_kmer_count_canonical": ("base starts lut hist status", lambda a: ops.rows_kmer_count_canonical(
        *_rows(a), nv.ENC_LUT, 5, 3, BINS, a["lut"], a["hist"], status=a["status"])),
    "rows_kmer_table_insert": ("base starts lut keys status", lambda a: ops.rows_kmer_table_insert(
        *_rows(a), nv.ENC_LUT, 5, a["keys"], a["counts"], a["n_used"], 0, a["lut"], a["status"])),
    "kmer_table_rehash": ("keys new_keys status", lambda a: ops.kmer_table_rehash(
        a["keys"], a["counts"], a["new_keys"], a["new_counts"], a["n_used"], a["status"])),
    "rows_pwm_scores": ("base starts lut matrix offsets status", lambda a: ops.rows_pwm_scores(
        *_rows(a), nv.ENC_LUT, a["matrix"], a["lut"], False, a["offsets"], a["status"], a["total"])),
    "rows_pwm_max": ("base starts lut matrix status", lambda a: ops.rows_pwm_max(
        *_rows(a), nv.ENC_LUT, a["matrix"], a["lut"], a["status"])),
    "rows_match": ("base starts lut sets offsets status out", lambda a: ops.rows_match(
        *_rows(a), nv.ENC_LUT, 4, a["sets"], [2], False, a["lut"], a["offsets"], a["status"], a["total"], a["out"])),
    "rows_match_count": ("base starts lut sets status", lambda a: ops.rows_match_count(
        *_rows(a), nv.ENC_LUT, 4, a["sets"], [2], False, a["lut"], a["status"])),
    "bincount": ("values hist status", lambda a: ops.bincount(a["values"], BINS, a["hist"], status=a["status"])),
    "bincount_rows": ("values row_bounds status", lambda a: ops.bincount_rows(
        a["values"], a["row_bounds"], 4, a["status"])),
    "synth_fastq": ("synth_out", lambda a: ops.synth_fastq(2, out=a["synth_out"])),
    "HostPipeline.kmer_count": ("hist lut_host chunk_host", lambda a: a["pipeline"].kmer_count(
        a["chunk_host"], 5, a["hist"], enc_mode=nv.ENC_LUT, lut_host=a["lut_host"])),
    "multiline_flags": ("fasta f_starts", lambda a: ops.multiline_flags(a["fasta"], a["f_starts"], a["f_lens"])),
    "multiline_entries": ("fasta f_starts is_header hdr_before", lambda a: ops.multiline_entries(
        a["fasta"], a["f_starts"], a["f_lens"], a["is_header"], a["hdr_before"], 2, False)),
    "bloom_insert": ("values hash_offsets mask", lambda a: ops.bloom_insert(a["values"], a["hash_offsets"], a["mask"])),
    "bloom_query": ("values hash_offsets mask", lambda a: ops.bloom_query(a["values"], a["hash_offsets"], a["mask"])),
    "reset_status": ("status", lambda a: ops.reset_status(a["status"])),
    "format_offsets": ("base starts lut status", lambda a: ops.format_offsets(
        nv.FMT_FASTA, 1, _fields(a), a["status"])),
    "format_records": ("base starts lut rec_offsets text_out", lambda a: ops.format_records(
        nv.FMT_FASTA, 1, _fields(a), a["rec_offsets"], 0, 8, a["text_out"])),
    "delimited_columns": ("bed b_starts status", lambda a: ops.delimited_columns(
        a["bed"], a["b_starts"], a["b_lens"], [nv.COL_TEXT, nv.COL_INT, nv.COL_STRAND], a["status"])),
    "name_lookup": ("base starts name_table name_offsets status", lambda a: ops.name_lookup(
        *_rows(a), a["name_table"], a["name_offsets"], a["status"])),
    "interval_check": ("base start stop status", lambda a: ops.interval_check(
        a["base"], a["start"], a["stop"], status=a["status"])),
    "interval_copy": ("base start stop iv_offsets strand lut", lambda a: ops.interval_copy(
        a["base"], a["start"], a["stop"], a["iv_offsets"], 12, strand=a["strand"], complement_lut=a["lut"])),
    "interval_events": ("start stop status", lambda a: ops.interval_events(
        a["start"], a["stop"], size=10, glob=True, status=a["status"])),
    "pileup_runs": ("sorted_keys", lambda a: ops.pileup_runs(a["sorted_keys"], 10)),
    "runs_reduce": ("run_starts run_values q_start stop", lambda a: ops.runs_reduce(
        a["run_starts"], a["run_values"], a["q_start"], a["stop"], nv.RUNS_MAX)),
    "runs_extract": ("run_starts run_values q_start out_offsets", lambda a: ops.runs_extract(
        a["run_starts"], a["run_values"], a["q_start"], a["out_offsets"], 4)),
    "interval_merge": ("start stop same_prev status", lambda a: ops.interval_merge(
        a["start"], a["stop"], a["same_prev"], 0, a["status"])),
    "rows_equal_prev": ("base starts", lambda a: ops.rows_equal_prev(*_rows(a))),
    "runs_combine": ("run_starts run_values", lambda a: ops.runs_combine(
        a["run_starts"], a["run_values"], a["run_starts"].clone(), a["run_values"].clone(), nv.OP_ADD)),
    "interval_intersect": ("start stop same_prev", lambda a: ops.interval_intersect(a["start"], a["stop"],
                                                                                    a["same_prev"])),
    "runs_to_intervals": ("run_starts run_values contig_ends", lambda a: ops.runs_to_intervals(
        a["run_starts"], a["run_values"], a["contig_ends"])),
    "delimited_offsets": ("values strand_col status", lambda a: ops.delimited_offsets(_columns(a), a["status"])),
    "delimited_format": ("values strand_col line_offsets text_out", lambda a: ops.delimited_format(
        _columns(a), a["line_offsets"], 0, 8, a["text_out"])),
}


def _cpu(t):
    return t.cpu()


def _cuda(t):
    return t.to(DEV)


def _short(t):
    return t[:-1]


def _int64(t):
    return t.long()


def _int32(t):
    return t.int()


def _strided(t):
    return torch.stack([t, t], 1)[:, 0]


OFFSETS = [(_cpu, nv.NativeLibraryError), (_short, ValueError)]
# argument -> the ways the cases make it wrong and what each raises
BAD = {"lut": [(_cpu, nv.NativeLibraryError), (_short, TypeError), (_int64, TypeError)],
       "offsets": OFFSETS, "rec_offsets": OFFSETS, "line_offsets": OFFSETS, "iv_offsets": OFFSETS,
       "out_offsets": OFFSETS, "hdr_before": OFFSETS, "name_offsets": [(_int32, TypeError)],
       "row_bounds": [(_cpu, nv.NativeLibraryError), (_int32, TypeError)],
       "hist": [(_int32, TypeError), (_short, ValueError)],
       "status": [(_short, ValueError), (_cpu, nv.NativeLibraryError)],
       "out": [(_cpu, nv.NativeLibraryError), (_short, ValueError)], "text_out": [(_cpu, nv.NativeLibraryError)],
       "synth_out": [(_cpu, nv.NativeLibraryError), (_short, ValueError)],
       "base": [(_strided, ValueError)], "fasta": [(_strided, ValueError)], "bed": [(_strided, ValueError)],
       "starts": [(_short, ValueError)], "f_starts": [(_short, ValueError)], "b_starts": [(_short, ValueError)],
       "stop": [(_short, ValueError)], "is_header": [(_short, ValueError)], "same_prev": [(_int64, ValueError)],
       "keys": [(_short, ValueError)], "new_keys": [(_short, ValueError)], "matrix": [(_cpu, nv.NativeLibraryError)],
       "sets": [(_int64, TypeError)], "strand": [(_short, ValueError)], "strand_col": [(_short, ValueError)],
       "values": [(_int32, TypeError)],
       "run_values": [(_short, ValueError)], "contig_ends": [(_cpu, nv.NativeLibraryError)],
       "mask": [(_int64, TypeError)], "hash_offsets": [(_int32, TypeError)], "sorted_keys": [(_int32, TypeError)],
       "lut_host": [(_cuda, TypeError), (_short, TypeError)], "chunk_host": [(_strided, ValueError)]}
BAD_FOR = {"HostPipeline.kmer_count": {"hist": [(_cpu, nv.NativeLibraryError), (_int32, TypeError)]}}


def _cases():
    cases = {}
    for op, (names, _) in OPS.items():
        names = names.split()
        first = [(names[0], _cpu, nv.NativeLibraryError)]
        bad_for = {**BAD, **BAD_FOR.get(op, {})}
        for name, bad, exc in first + [(n, b, e) for n in names for b, e in bad_for.get(n, [])]:
            cases.setdefault(f"{op}-{name}-{bad.__name__[1:]}", (op, name, bad, exc))
    return cases


CASES = _cases()


@pytest.mark.parametrize("op", list(OPS))
def test_valid_arguments_launch(op):
    """The arguments the rejections below start from are accepted, and the op launches its kernels."""
    a = _valid(op)
    lib = nv.load_library()
    before = lib.bnpk_launch_count()
    OPS[op][1](a)
    torch.cuda.synchronize()
    assert lib.bnpk_launch_count() > before


class _NoLibrary:
    """Stands in for libbnpk.so while a rejected call runs: any call of it fails the test."""

    def __getattr__(self, name):
        def called(*args):
            pytest.fail(f"a rejected argument reached {name}")
        return called


@pytest.mark.parametrize("case", list(CASES))
def test_rejected_argument_launches_nothing(case, monkeypatch):
    op, name, bad, exc = CASES[case]
    a = _valid(op)
    a[name] = bad(a[name])
    torch.cuda.synchronize()
    before = nv.load_library().bnpk_launch_count()
    monkeypatch.setattr(ops, "lib", lambda: _NoLibrary())
    with pytest.raises(exc):
        OPS[op][1](a)
    assert nv.load_library().bnpk_launch_count() == before


def test_argument_error_is_both_a_type_and_a_value_error():
    """A wrong dtype or element count raises ops.ArgumentError, which callers may catch as TypeError or ValueError."""
    lut = torch.zeros(255, dtype=torch.uint8, device=DEV)
    base, starts, lens = _view(ROWS)
    for err in (TypeError, ValueError, ops.ArgumentError):
        with pytest.raises(err):
            ops.rows_reverse_complement(base, starts, lens, lut)
