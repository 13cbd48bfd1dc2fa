"""The torch.ops.bnpk binding checks every tensor a kernel would read before it launches anything: a CPU or short lut,
CPU or short offsets, starts and lens of different lengths, a wrong dtype and canonical minimizers all raise, and
bnpk_launch_count() stays where it was.  The writer ops give the same bytes as ops.format_*."""
import numpy as np
import pytest
import torch

from bionumpy_b200 import _native as nv
from bionumpy_b200 import ops, torch_ops

pytestmark = pytest.mark.gpu
DEV = "cuda"
ROWS = [b"ACGTACGTTGCA", b"GGGCCCAATT", b"TTTTACGTAGCTAGCT"]
NAMES = [b"r0", b"r1", b"r2"]


def _view(rows):
    """(base uint8, starts int64, lens int32) of the rows laid end to end on the device."""
    lens = [len(r) for r in rows]
    starts = np.concatenate([[0], np.cumsum(lens)[:-1]]).astype(np.int64)
    base = np.frombuffer(b"".join(rows), dtype=np.uint8).copy()
    return (torch.from_numpy(base).to(DEV), torch.from_numpy(starts).to(DEV),
            torch.tensor(lens, dtype=torch.int32, device=DEV))


def _dna_lut():
    t = np.full(256, 255, dtype=np.uint8)
    for c, v in zip(b"ACGT", range(4)):
        t[c] = v
    return torch.from_numpy(t).to(DEV)


def _letters():
    """The output table of ACGT codes: code c -> b"ACGT"[c], other codes 0 (a bad code)."""
    t = torch.zeros(256, dtype=torch.uint8, device=DEV)
    t[:4] = torch.tensor(list(b"ACGT"), dtype=torch.uint8)
    return t


def _args():
    """Valid arguments of every row op: the rows, an ENC_LUT table, offsets int64[R + 1] and the output total."""
    base, starts, lens = _view(ROWS)
    offsets = torch.zeros(len(ROWS) + 1, dtype=torch.int64, device=DEV)
    offsets[1:] = torch.cumsum(lens.long(), 0)
    return dict(base=base, starts=starts, lens=lens, enc=nv.ENC_LUT, lut=_dna_lut(), offsets=offsets,
                total=int(offsets[-1]), window=0, cxor=0)


def _call(op, a):
    top = torch_ops.load()
    rows = (a["base"], a["starts"], a["lens"])
    if op == "rows_encode":
        return top.rows_encode(*rows, a["enc"], a["lut"], a["offsets"], a["total"])
    if op == "rows_kmer_hash":
        return top.rows_kmer_hash(*rows, a["enc"], a["lut"], 5, a["window"], a["cxor"], a["offsets"], a["total"])
    if op == "rows_kmer_count":
        hist = torch.zeros(1024, dtype=torch.int64, device=DEV)
        return top.rows_kmer_count(*rows, a["enc"], a["lut"], 5, a["window"], a["cxor"], hist)
    if op == "rows_kmer_table_insert":
        keys = torch.full((1024,), -1, dtype=torch.int64, device=DEV)
        counts = torch.zeros(1024, dtype=torch.int64, device=DEV)
        n_used = torch.zeros(1, dtype=torch.int64, device=DEV)
        return top.rows_kmer_table_insert(*rows, a["enc"], a["lut"], 5, a["cxor"], keys, counts, n_used)
    if op == "rows_reverse_complement":
        return top.rows_reverse_complement(*rows, a["lut"], a["offsets"], a["total"])
    if op == "rows_pwm_scores":
        matrix = torch.ones(3, 4, dtype=torch.float64, device=DEV)
        return top.rows_pwm_scores(*rows, a["enc"], a["lut"], matrix, False, a["offsets"], a["total"])
    if op == "rows_match":
        sets = torch.tensor([1, 2], dtype=torch.int32, device=DEV)          # "AC"
        return top.rows_match(*rows, a["enc"], a["lut"], 4, sets, [2], False, a["offsets"], a["total"])
    if op == "chunk_kmer_count":
        chunk = torch.from_numpy(np.frombuffer(b"@r\nACGTACGT\n+\nIIIIIIII\n", dtype=np.uint8).copy()).to(DEV)
        hist = torch.zeros(1024, dtype=torch.int64, device=DEV)
        return top.chunk_kmer_count(chunk, 5, 0, hist, 4, ord("@"), True, -1, a["enc"], a["lut"])
    fields = list(_view(NAMES)) + [a["base"], a["starts"], a["lens"]]
    luts = [None, a["lut"]]
    if op == "format_offsets":
        return top.format_offsets(nv.FMT_FASTA, 1, fields, luts)
    assert op == "format_records"
    return top.format_records(nv.FMT_FASTA, 1, fields, luts, a["offsets"], 0, 4)


def _as_fasta_records(a):
    """format ops: the rows are the sequences of FASTA records named NAMES, held as codes 0..3 under an output table
    back to letters; offsets are the records' output offsets."""
    a["base"] = _dna_lut()[a["base"].long()]
    a["lut"] = _letters()
    sizes = [len(b">\n\n") + len(n) + len(r) for n, r in zip(NAMES, ROWS)]
    a["offsets"] = torch.tensor(np.concatenate([[0], np.cumsum(sizes)]), dtype=torch.int64, device=DEV)


LUT_OPS = ["rows_encode", "rows_kmer_hash", "rows_kmer_count", "rows_kmer_table_insert", "rows_reverse_complement",
           "rows_pwm_scores", "rows_match", "chunk_kmer_count", "format_offsets", "format_records"]
OFFSET_OPS = ["rows_encode", "rows_kmer_hash", "rows_reverse_complement", "rows_pwm_scores", "rows_match",
              "format_records"]
ROW_OPS = [op for op in LUT_OPS if op != "chunk_kmer_count"]


def _cpu_lut(a):
    a["lut"] = a["lut"].cpu()


def _lut_255(a):
    a["lut"] = a["lut"][:255]


def _cpu_offsets(a):
    a["offsets"] = a["offsets"].cpu()


def _short_offsets(a):
    a["offsets"] = a["offsets"][:len(ROWS)]


def _short_starts(a):
    a["starts"] = a["starts"][:-1]


def _lens_int64(a):
    a["lens"] = a["lens"].long()


def _minimizer_cxor(a):
    a["window"], a["cxor"] = 7, 3


CASES = ([(op, _cpu_lut) for op in LUT_OPS] + [(op, _lut_255) for op in LUT_OPS] +
         [(op, _cpu_offsets) for op in OFFSET_OPS] + [(op, _short_offsets) for op in OFFSET_OPS] +
         [(op, _short_starts) for op in ROW_OPS] + [(op, _lens_int64) for op in ROW_OPS] +
         [(op, _minimizer_cxor) for op in ("rows_kmer_hash", "rows_kmer_count")])


def _valid(op):
    a = _args()
    if op.startswith("format_"):
        _as_fasta_records(a)
    return a


@pytest.mark.parametrize("op", LUT_OPS)
def test_valid_arguments_launch(op):
    """The arguments the rejections below start from are accepted, and the op launches its kernels."""
    lib = nv.load_library()
    before = lib.bnpk_launch_count()
    _call(op, _valid(op))
    torch.cuda.synchronize()
    assert lib.bnpk_launch_count() > before


@pytest.mark.parametrize("op,bad", CASES, ids=[f"{op}-{bad.__name__[1:]}" for op, bad in CASES])
def test_rejected_argument_launches_nothing(op, bad):
    lib = nv.load_library()
    a = _valid(op)
    bad(a)
    before = lib.bnpk_launch_count()
    with pytest.raises(RuntimeError):
        _call(op, a)
    assert lib.bnpk_launch_count() == before


def _fields(rng, n, codes):
    """(name, sequence, quality) fields of n random records for ops.format_*, the sequence as codes with an output
    table back to letters when `codes`."""
    names = [bytes(rng.integers(33, 127, int(rng.integers(0, 12)), dtype=np.uint8)) for _ in range(n)]
    seq_lens = rng.integers(0, 300, n)
    seqs = [bytes(rng.integers(0, 4, int(m), dtype=np.uint8)) for m in seq_lens]
    if not codes:
        seqs = [bytes(b"ACGT"[c] for c in s) for s in seqs]
    quals = [bytes(rng.integers(33, 127, int(m), dtype=np.uint8)) for m in seq_lens]
    return (_view(names) + (None,), _view(seqs) + (_letters() if codes else None,), _view(quals) + (None,))


@pytest.mark.parametrize("fmt,width,codes", [(nv.FMT_FASTQ, 1, False), (nv.FMT_FASTA_WRAPPED, 60, True),
                                             (nv.FMT_FASTA_WRAPPED, 7, False)])
def test_format_ops_match_ctypes_ops(fmt, width, codes):
    top = torch_ops.load()
    fields = _fields(np.random.default_rng(width), 500, codes)
    if fmt != nv.FMT_FASTQ:
        fields = fields[:2] + (None,)
    want_offsets, want_status = ops.format_offsets(fmt, width, fields)
    want = ops.format_records(fmt, width, fields, want_offsets)
    used = [f for f in fields if f is not None]
    flat = [t for f in used for t in f[:3]]
    luts = [f[3] for f in used]
    offsets, status = top.format_offsets(fmt, width, flat, luts)
    assert torch.equal(offsets, want_offsets)
    assert torch.equal(status, want_status)
    total = int(offsets[-1])
    got = top.format_records(fmt, width, flat, luts, offsets, 0, total)
    assert total > 0 and torch.equal(got, want)
    part = top.format_records(fmt, width, flat, luts, offsets, 5, total - 3)
    assert torch.equal(part, want[5:total - 3])
