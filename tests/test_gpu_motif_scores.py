"""Motif scores (K7, row_kernels.cu) against the NumPy restatement of the reference, bit for bit.

Scores are compared as int64 bit patterns, so -inf, +0.0 and every last bit count.  NaN (a +inf and a -inf column in
one window) is compared by position only: the GPU's inf - inf is its canonical NaN, x86's is a NaN of another payload.

Rows are walked in 2 KiB staging segments by the four-letter kernels: the first segment holds 2048 - off bytes (off =
the address of the row's first byte mod 16), and each later one starts m - 1 bytes before the previous one ends.  Row
lengths sit at -1, 0 and +1 around the first two segment edges for every address mod 16, the view starts at byte 0..15
of an aligned allocation, and every byte no row covers is poison, so a read past a row changes a score or reports a bad
byte.  The segment rule is restated only to place the lengths; the oracle decides what is correct."""
import gzip
import os
from collections import namedtuple

import numpy as np
import pytest
import torch

import bionumpy_b200 as bnp
from bionumpy_b200 import _native as nv
from bionumpy_b200 import ops
from bionumpy_b200.encodings.exceptions import EncodingError
from bionumpy_b200.sequence.position_weight_matrix import PWM, PositionWeightMatrix
from oracle import bnp_oracle as o

import motif_oracle as mo

gpu = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
SEG = 2048
AMINO = "ACDEFGHIKLMNPQRSTVWY*"
MOTIF_LENS = [1, 2, 6, 16, 31, 32, 33, 64, 100, 1024]

# mode / lut: what the kernel is given; table: the oracle's byte -> code table (255 = invalid); letters: the bytes rows
# are drawn from; poison: a byte outside the alphabet
Enc = namedtuple("Enc", "mode lut table size letters poison")


def _text(alphabet, mode=nv.ENC_LUT):
    table = o.alphabet_lut(alphabet)
    letters = np.frombuffer((alphabet.replace("*", "") + alphabet.lower().replace("*", "")).encode(), dtype=np.uint8)
    return Enc(mode, table if mode == nv.ENC_LUT else None, table, len(alphabet), letters, ord("X"))


def _codes(size):
    table = np.full(256, 255, dtype=np.uint8)
    table[:size] = np.arange(size)
    return Enc(nv.ENC_CODES, None, table, size, np.arange(size, dtype=np.uint8), 200)


ENCODINGS = {
    "acgt": _text("ACGT", nv.ENC_ASCII_ACGT),
    "actg": _text("ACTG", nv.ENC_ASCII_ACTG),
    "codes": _codes(4),
    "lut_tgca": _text("TGCA"),
    "ace": _text("ACE"),
    "acgtn": _text("ACGTN"),
    "amino": _text(AMINO),
    "amino_codes": _codes(21),
}


def assert_bits(got, want):
    got = got.detach().cpu().numpy() if isinstance(got, torch.Tensor) else np.asarray(got)
    want = np.asarray(want, dtype=np.float64)
    assert got.dtype == np.float64 and got.shape == want.shape, (got.shape, want.shape)
    gn, wn = np.isnan(got), np.isnan(want)
    assert np.array_equal(gn, wn), np.flatnonzero(gn != wn)[:10]
    bad = np.flatnonzero(got[~gn].view(np.int64) != want[~wn].view(np.int64))
    assert bad.size == 0, (bad[:10], got[~gn][bad[:5]], want[~wn][bad[:5]])


def random_matrix(rng, size, m, infs=False):
    mat = rng.normal(0.0, 1.7, size=(size, m)) + rng.random((size, m)) * 1e-3
    if infs:
        mat[rng.integers(0, size, m // 3 + 1), rng.integers(0, m, m // 3 + 1)] = -np.inf
        mat[rng.integers(0, size, 2), rng.integers(0, m, 2)] = np.inf
    return mat


def edge_lengths(m):
    """(address mod 16, length) pairs: -1/0/+1 around the first two segment edges, plus 0, 1, m - 1, m, m + 1."""
    out = []
    for off0 in range(16):
        end1 = SEG - off0
        s2 = end1 - (m - 1)
        end2 = s2 + SEG - (off0 + s2) % 16
        for e in (end1, end2):
            out += [(off0, e + d) for d in (-1, 0, 1)]
    out += [(int(i), L) for i, L in enumerate((0, 1, max(m - 1, 0), m, m + 1, 2 * m + 5))]
    return out


class View:
    """Rows in one aligned device allocation, seen from byte `view_off`; poison everywhere else."""

    def __init__(self, rng, enc, placements, view_off):
        total = view_off + sum(L + 40 for _, L in placements) + 64
        buf = np.full(total, enc.poison, dtype=np.uint8)
        starts, lens, pos = [], [], view_off + 8
        for off0, L in placements:
            pos += (off0 - pos) % 16
            buf[pos:pos + L] = rng.choice(enc.letters, size=L)
            starts.append(pos - view_off)
            lens.append(L)
            pos += L + int(rng.integers(1, 24))
        self.host = buf[view_off:]
        dev = torch.from_numpy(buf).cuda()
        assert dev.data_ptr() % 256 == 0
        self.base = dev[view_off:]
        self.starts = torch.tensor(starts, dtype=torch.int64, device="cuda")
        self.lens = torch.tensor(lens, dtype=torch.int32, device="cuda")
        self.rows = [self.host[s:s + L] for s, L in zip(starts, lens)]

    def codes(self, enc):
        flat = np.concatenate(self.rows) if self.rows else np.zeros(0, np.uint8)
        c = enc.table[flat]
        assert (c != 255).all()
        return c.astype(np.int64), np.array([len(r) for r in self.rows])


def _run(view, enc, mat):
    dev_mat = torch.from_numpy(np.ascontiguousarray(mat.T)).cuda()
    lut = torch.from_numpy(enc.lut).cuda() if enc.lut is not None else None
    scores, offsets, st = ops.rows_pwm_scores(view.base, view.starts, view.lens, enc.mode, dev_mat, lut)
    tail, _, st_t = ops.rows_pwm_scores(view.base, view.starts, view.lens, enc.mode, dev_mat, lut, tail=True)
    best, st_m = ops.rows_pwm_max(view.base, view.starts, view.lens, enc.mode, dev_mat, lut)
    return scores, tail, best, [ops.read_status(s) for s in (st, st_t, st_m)]


def _cases():
    for name in ENCODINGS:
        for m in MOTIF_LENS:
            if ENCODINGS[name].size * m > 8192:
                m = 8192 // ENCODINGS[name].size
            yield pytest.param(name, m, id=f"{name}-m{m}")


@gpu
@pytest.mark.parametrize("enc_name,m", list(_cases()))
def test_rows_against_oracle(enc_name, m):
    enc = ENCODINGS[enc_name]
    rng = np.random.default_rng(m * 31 + len(enc_name))
    view = View(rng, enc, edge_lengths(m), int(rng.integers(0, 16)))
    codes, lens = view.codes(enc)
    for infs in (False, True):
        mat = random_matrix(rng, enc.size, m, infs)
        scores, tail, best, sts = _run(view, enc, mat)
        want, want_lens = mo.motif_scores(codes, lens, mat)
        assert_bits(scores, want)
        assert_bits(best, mo.row_max(want, want_lens))
        pos = np.concatenate([[0], np.cumsum(lens)])
        want_tail = np.concatenate([mo.calculate_scores(codes[pos[i]:pos[i + 1]], mat) for i in range(len(lens))])
        assert_bits(tail, want_tail)
        for st in sts:
            assert st.bad_base() is None and st.n_bases == int(lens.sum())
        assert sts[0].n_values == want.size == sts[2].n_values and sts[1].n_values == int(lens.sum())


@gpu
@pytest.mark.parametrize("view_off", range(16))
def test_every_view_offset(view_off):
    enc = ENCODINGS["acgt"]
    rng = np.random.default_rng(view_off)
    m = 33
    view = View(rng, enc, edge_lengths(m), view_off)
    codes, lens = view.codes(enc)
    mat = random_matrix(rng, 4, m)
    scores, tail, best, _ = _run(view, enc, mat)
    want, want_lens = mo.motif_scores(codes, lens, mat)
    assert_bits(scores, want)
    assert_bits(best, mo.row_max(want, want_lens))


# -- public API ------------------------------------------------------------------------------------------------------
DOC_DICT = {"A": [5, 1], "C": [1, 5], "G": [0, 0], "T": [0, 0]}
TEST_MATRIX = np.log([[0.4, 0.25], [0.1, 0.25], [0.4, 0.25], [0.1, 0.25]])


@gpu
def test_reference_goldens():
    pwm = PWM.from_dict(DOC_DICT)
    got = bnp.get_motif_scores(bnp.as_encoded_array(["ACTGAC", "CA", "GG"]), pwm)
    assert got.tolist() == [[5.991464547107982, -np.inf, -np.inf, -np.inf, 5.991464547107982], [2.772588722239781],
                            [-np.inf]]
    assert_bits(bnp.get_motif_scores(["ACTGAC", "CA", "GG"], pwm).max(axis=-1),
                [5.991464547107982, 2.772588722239781, -np.inf])
    a = PWM.from_dict({"A": [1, 1], "C": [0, 0], "G": [0, 0], "T": [0, 0]})
    assert_bits(a.calculate_scores("AAC"), [np.log(4 ** 2), -np.inf, -np.inf])
    neutral = PWM.from_dict({c: [0.25, 0.25] for c in "ACGT"})
    seq = bnp.EncodedArray(np.array([0, 1, 2, 3]), bnp.DNAEncoding)
    assert_bits(neutral.calculate_scores(seq), [0.0, 0.0, 0.0, 0.0])
    pwm = PWM(TEST_MATRIX, "ACGT")
    window = bnp.EncodedArray(np.array([0, 1]), bnp.DNAEncoding)
    assert np.isclose(np.exp(PositionWeightMatrix(pwm)(window)), 0.1)
    assert np.isclose(np.exp(pwm.calculate_score(window)), 0.1)
    assert np.allclose(np.exp(PositionWeightMatrix(pwm).rolling_window(seq).cpu().numpy()), [0.1, 0.025, 0.1])
    seqs = ["ACGT", "GCT"]
    assert PositionWeightMatrix(pwm).rolling_window(seqs).tolist() == bnp.get_motif_scores(seqs, pwm).tolist()
    assert_bits(bnp.get_motif_scores("ACGTAC", pwm), mo.calculate_scores(mo.encode([b"ACGTAC"], "ACGT")[0],
                                                                        TEST_MATRIX)[:5])


@gpu
@pytest.mark.parametrize("alphabet", ["ACGT", "TGCA", "ACE"])
def test_nan_propagates_to_the_row_maximum(alphabet):
    """+inf in column 0 and -inf in column 1: a window starting with those two letters scores NaN, and np.max makes
    its row's maximum NaN (fmax would not)."""
    mat = np.zeros((len(alphabet), 3))
    mat[0, 0], mat[1, 1], mat[2, 2] = np.inf, -np.inf, 2.5
    pwm = PWM(mat, alphabet)
    a, b, c = alphabet[:3]
    rows = [c * 5 + a + b + c * 5, a + b, c * 6, b + a + a]
    want_codes, _ = mo.encode([r.encode() for r in rows], alphabet)
    want, want_lens = mo.motif_scores(want_codes, [len(r) for r in rows], mat)
    best = bnp.get_motif_scores(rows, pwm).max(axis=-1)
    assert np.isnan(best[0].item()) and best[1].item() == -np.inf and best[2].item() == 2.5
    assert_bits(best, mo.row_max(want, want_lens))
    assert_bits(bnp.get_motif_scores(rows, pwm).ravel(), want)


@gpu
def test_calculate_score_long_motif_is_close_to_the_pairwise_sum():
    rng = np.random.default_rng(5)
    mat = random_matrix(rng, 4, 40)
    pwm = PWM(mat, "ACGT")
    codes = rng.integers(0, 4, 40)
    got = pwm.calculate_score(bnp.EncodedArray(codes, bnp.DNAEncoding))
    assert got == mo.calculate_scores(codes, mat)[0]                     # column order, bit for bit
    assert np.isclose(got, mat[codes, np.arange(40)].sum(), rtol=1e-12, atol=0)


def _api_inputs(rng, alphabet, lens, encoded=None):
    letters = alphabet.replace("*", "")
    rows = ["".join(rng.choice(list(letters + letters.lower()), size=L)) for L in lens]
    codes, _ = mo.encode([r.encode() for r in rows], alphabet)
    if encoded is not None:
        seq = bnp.as_encoded_array([r.upper() for r in rows], encoded)
    else:
        seq = bnp.as_encoded_array(rows)
    return seq, codes


@gpu
@pytest.mark.parametrize("alphabet,encoded", [("ACGT", None), ("ACTG", None), ("ACGT", bnp.DNAEncoding),
                                              ("TGCA", None), ("ACE", None), ("ACGTN", None),
                                              ("ACGTN", bnp.AlphabetEncoding("ACGTN")), (AMINO, None),
                                              (AMINO, bnp.AminoAcidEncoding)])
@pytest.mark.parametrize("m", [1, 6, 33])
def test_api_alphabets_and_split_rows(alphabet, encoded, m):
    """Every route through get_motif_scores, with a row long enough to be cut into pieces (> 2^14 windows)."""
    rng = np.random.default_rng(len(alphabet) * 100 + m)
    lens = [0, 3, m - 1, m, 150, 40000, 17, 2100]
    seq, codes = _api_inputs(rng, alphabet, lens, encoded)
    mat = random_matrix(rng, len(alphabet), m, infs=m == 6)
    pwm = PWM(mat, alphabet)
    want, want_lens = mo.motif_scores(codes, lens, mat)
    got = bnp.get_motif_scores(seq, pwm)
    assert got.lengths.cpu().tolist() == want_lens.tolist()
    best = bnp.get_motif_scores(seq, pwm).max(axis=-1)                   # fused, pieces combined on the device
    assert_bits(got.ravel(), want)
    assert_bits(best, mo.row_max(want, want_lens))
    assert_bits(got.max(axis=-1), mo.row_max(want, want_lens))         # materialised
    flat = np.concatenate([codes])
    assert_bits(pwm.calculate_scores(seq), mo.calculate_scores(flat, mat))
    hits = got > 0.5
    assert hits.ravel().cpu().numpy().tolist() == (want > 0.5).tolist()


@gpu
def test_encoded_alphabet_longer_than_the_pwm():
    rng = np.random.default_rng(3)
    pwm = PWM(random_matrix(rng, 4, 5), "ACGT")
    enc = bnp.AlphabetEncoding("ACGTN")
    ok = bnp.as_encoded_array(["ACGTACGTTT", "GGA"], enc)
    codes = np.array([0, 1, 2, 3, 0, 1, 2, 3, 3, 3, 2, 2, 0])
    want, lens = mo.motif_scores(codes, [10, 3], pwm._matrix)
    assert_bits(bnp.get_motif_scores(ok, pwm).ravel(), want)
    with pytest.raises(Exception, match=r"Could not calculate pwm for alphabet \['A', 'C', 'G', 'T'\] on "
                                        r"\['A', 'C', 'G', 'T', 'N'\] encoded array"):
        bnp.get_motif_scores(bnp.as_encoded_array(["ACGTN"], enc), pwm)
    with pytest.raises(Exception, match="Could not calculate pwm"):
        bnp.get_motif_scores(bnp.as_encoded_array(["ACGT"], bnp.ACTGEncoding), pwm)


@gpu
@pytest.mark.parametrize("alphabet", ["ACGT", "ACTG", "TGCA", "ACE", "ACGTN"])
@pytest.mark.parametrize("where", ["first", "interior", "last", "overlap", "tail", "split_piece"])
def test_bad_bytes(alphabet, where):
    """EncodingError.offset is the oracle's first bad flat offset, for the materialised scores, the fused maximum and
    calculate_scores."""
    m = 12
    rng = np.random.default_rng(sum(map(ord, alphabet + where)))
    lens = [30, 5000 if where != "split_piece" else 40000, 9]
    L = lens[1]
    pos = {"first": 3, "interior": 1000, "last": L - 1, "overlap": SEG - 16 - 4,
           "tail": L - 5, "split_piece": 30000}[where]
    letters = alphabet
    rows = ["".join(rng.choice(list(letters), size=n)) for n in lens]
    rows[1] = rows[1][:pos] + "x" + rows[1][pos + 1:]
    want = lens[0] + pos
    _, bad = mo.encode([r.encode() for r in rows], alphabet)
    assert bad == want
    pwm = PWM(random_matrix(rng, len(alphabet), m), alphabet)
    for fn in (lambda: bnp.get_motif_scores(rows, pwm).ravel(), lambda: bnp.get_motif_scores(rows, pwm).max(axis=-1),
               lambda: pwm.calculate_scores(rows)):
        with pytest.raises(EncodingError) as e:
            fn()
        assert e.value.offset == want


@gpu
def test_fused_max_writes_no_scores(big_fq_path):
    """The reference's pwm_example: scores of every read of big.fq.gz, and the per-read maximum by the fused kernel,
    which launches the max mode only (no score kernel) and leaves the lazy scores unmaterialised."""
    pwm = bnp.io.read_motif(os.path.join(GOLDEN, "MA0080.1.jaspar"))
    seq = bnp.open(big_fq_path).read().sequence
    raw = seq.ravel().raw().cpu().numpy()
    codes, bad = mo.encode([raw.tobytes()], "ACGT")
    assert bad is None
    lens = seq.lengths.cpu().numpy()
    want, want_lens = mo.motif_scores(codes, lens, pwm._matrix)
    lazy = bnp.get_motif_scores(seq, pwm)
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        best = lazy.max(axis=-1)
        torch.cuda.synchronize()
    names = [e.name for e in prof.events() if "bnpk::rows_" in e.name]
    assert names and all("rows_pwm_kernel<7" in n for n in names), set(names)     # RM_PWM_MAX only
    assert not lazy.is_materialised()
    assert_bits(best, mo.row_max(want, want_lens))
    assert_bits(lazy.ravel(), want)
    chunks = [c.sequence for c in bnp.open(big_fq_path).read_chunks(50000)]
    assert len(chunks) > 1
    got = torch.cat([bnp.get_motif_scores(c, pwm).max(axis=-1) for c in chunks])
    assert_bits(got, mo.row_max(want, want_lens))


@gpu
def test_sacCer3_whole_genome(tmp_path):
    raw = gzip.open(os.path.join(GOLDEN, "sacCer3.fa.gz")).read()
    path = tmp_path / "sacCer3.fa"
    path.write_bytes(raw)
    whole = np.frombuffer((raw if raw.endswith(b"\n") else raw + b"\n") + b">", dtype=np.uint8)
    _, _, _, flat, seq_lens = o.multiline_fasta_split(whole)
    codes = o.encode_flat(flat, o.alphabet_lut("ACGT")).astype(np.int64)
    seq = bnp.open(str(path)).read().sequence
    assert len(seq) == 17 and seq.lengths.cpu().numpy().tolist() == np.asarray(seq_lens).tolist()
    rng = np.random.default_rng(30)
    for pwm in (bnp.io.read_motif(os.path.join(GOLDEN, "MA0080.1.jaspar")), PWM(random_matrix(rng, 4, 30), "ACGT")):
        want, want_lens = mo.motif_scores(codes, seq_lens, pwm._matrix)
        assert_bits(bnp.get_motif_scores(seq, pwm).max(axis=-1), mo.row_max(want, want_lens))
        assert_bits(bnp.get_motif_scores(seq, pwm).ravel(), want)


@gpu
def test_two_streams_and_the_dispatcher_op():
    from bionumpy_b200 import torch_ops
    top = torch_ops.load()
    rng = np.random.default_rng(11)
    enc = ENCODINGS["lut_tgca"]
    views = [View(rng, enc, edge_lengths(m), 3) for m in (6, 40)]
    mats = [random_matrix(rng, 4, m) for m in (6, 40)]
    lut = torch.from_numpy(enc.lut).cuda()
    streams = [torch.cuda.Stream(), torch.cuda.Stream()]
    outs = []
    for v, mat, s in zip(views, mats, streams):
        with torch.cuda.stream(s):
            dm = torch.from_numpy(np.ascontiguousarray(mat.T)).cuda()
            outs.append(ops.rows_pwm_scores(v.base, v.starts, v.lens, enc.mode, dm, lut)[:2] + (dm,))
    torch.cuda.synchronize()
    for v, mat, (scores, offsets, dm) in zip(views, mats, outs):
        codes, lens = v.codes(enc)
        want, _ = mo.motif_scores(codes, lens, mat)
        assert_bits(scores, want)
        got, status = top.rows_pwm_scores(v.base, v.starts, v.lens, enc.mode, lut, dm, False, offsets, int(offsets[-1]))
        assert_bits(got, want)
        assert ops.read_status(status).bad_base() is None
