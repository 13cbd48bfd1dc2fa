"""String and pattern matches (K8, row_kernels.cu) against Python's ``re``, every bool and every count.

The four-letter kernels walk rows in 2 KiB staging segments: the first holds 2048 - off bytes (off = the address of the
row's first byte mod 16), each later one starts span - 1 bytes before the previous one ends.  Row lengths sit at -1, 0
and +1 around the first two segment edges for every address mod 16, the view starts at byte 0..15 of an aligned
allocation, and every byte no row covers is poison made of the pattern's own bytes, so a read past a row shows up as a
false match.  The segment rule is restated only to place the lengths; the oracle decides what is correct."""
import gzip
import os
import random

import numpy as np
import pytest
import torch

import bionumpy_b200 as bnp
from bionumpy_b200 import ops
from bionumpy_b200.encoded_array import BaseEncoding, EncodedArray, EncodedRaggedArray
from bionumpy_b200.encodings.exceptions import EncodingError
from bionumpy_b200.sequence.string_matcher import FixedLenRegexMatcher, RegexMatcher, StringMatcher
from oracle import bnp_oracle as o

import match_oracle as mo

gpu = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
SEG = 2048
AMINO = "ACDEFGHIKLMNPQRSTVWY*"
LENS = [1, 2, 3, 15, 16, 17, 31, 32, 33, 64, 100, 1024]
T, F = True, False

# name -> (matcher encoding, alphabet the oracle validates in (None: raw bytes), letters rows are drawn from, codes)
ROUTES = {
    "raw": (BaseEncoding, None, "ACGTacgtN", False),
    "acgt_text": (bnp.DNAEncoding, "ACGT", "ACGTacgt", False),
    "actg_text": (bnp.AlphabetEncoding("ACTG"), "ACTG", "ACGTacgt", False),
    "dna_codes": (bnp.DNAEncoding, "ACGT", "ACGT", True),
    "lut_tgca": (bnp.AlphabetEncoding("TGCA"), "TGCA", "ACGTacgt", False),
    "acgtn": (bnp.AlphabetEncoding("ACGTN"), "ACGTN", "ACGTNacgtn", False),
    "amino_text": (bnp.AminoAcidEncoding, AMINO, AMINO + "acdefy", False),
    "amino_codes": (bnp.AminoAcidEncoding, AMINO, AMINO, True),
}


def _pattern_letters(route):
    return "ACDEFY" if route.startswith("amino") else "ACGT"


def _patterns(route, m):
    """(kind, pattern, literal, span) of length m: a literal, a class pattern, and for m >= 3 leading/trailing dots."""
    rng = random.Random(m * 7 + len(route))
    letters = _pattern_letters(route)
    lit = "".join(rng.choice(letters) for _ in range(m))
    out = [("literal", lit, True)]
    if m >= 2:
        cls = "[" + letters[:2] + "]" + lit[1:-1] + "[" + letters[1:3] + "]" if m >= 2 else lit
        out.append(("class", cls, False))
    if m >= 3:
        out.append(("dots", "." + lit[1:-1] + ".", False))
    return out


def _instance(pattern, literal, rng, letters):
    """One string the pattern matches (classes and dots filled at random), for planting."""
    if literal:
        return pattern
    out, i = [], 0
    while i < len(pattern):
        c = pattern[i]
        if c == "[":
            end = pattern.index("]", i)
            out.append(rng.choice(pattern[i + 1:end]))
            i = end + 1
            continue
        if c == "." and pattern.startswith(".{", i):
            end = pattern.index("}", i)
            a, b = pattern[i + 2:end].split(",")
            out.extend(rng.choice(letters) for _ in range(rng.randint(int(a or 0), int(b))))
            i = end + 1
            continue
        out.append(rng.choice(letters) if c == "." else c)
        i += 1
    return "".join(out)


def _row(n, pattern, literal, rng, letters):
    """n bytes: random letters with instances of the pattern planted densely."""
    parts, size = [], 0
    while size < n:
        s = _instance(pattern, literal, rng, letters) if rng.random() < 0.5 else \
            "".join(rng.choice(letters) for _ in range(rng.randint(1, 8)))
        parts.append(s)
        size += len(s)
    return "".join(parts)[:n].encode()


def edge_lengths(span):
    """Lengths -1/0/+1 around the first two segment edges for a row starting at off (mod 16)."""
    out = []
    for off in range(16):
        e1 = SEG - off
        off2 = (1 - span) % 16
        e2 = e1 - (span - 1) + SEG - off2
        out.append((off, [max(e1 + d, 0) for d in (-1, 0, 1)] + [max(e2 + d, 0) for d in (-1, 0, 1)] + [0, 1, span]))
    return out


class View:
    """Rows placed at chosen addresses mod 16 in one buffer of poison; the view starts at byte `shift`."""

    def __init__(self, rows, offs, poison, shift, codes_of=None):
        buf, starts = bytearray(), []
        for r, off in zip(rows, offs):
            buf += poison * 3
            while (len(buf) + shift) % 16 != off:
                buf += poison[:1]
            starts.append(len(buf))
            buf += r
        buf += poison * 3
        raw = np.frombuffer(bytes(buf), dtype=np.uint8)
        if codes_of is not None:
            raw = codes_of(raw)
        alloc = torch.zeros(len(raw) + 32, dtype=torch.uint8, device="cuda")
        self.base = alloc[shift:shift + len(raw)]
        self.base.copy_(torch.from_numpy(raw.copy()))
        self.starts = torch.tensor(starts, dtype=torch.int64, device="cuda")
        self.lens = torch.tensor([len(r) for r in rows], dtype=torch.int32, device="cuda")
        self.rows = rows

    def array(self, encoding):
        return EncodedRaggedArray(EncodedArray(self.base, encoding), self.lens, starts=self.starts)


def _codes_of(alphabet):
    table = np.full(256, 255, dtype=np.uint8)
    for i, c in enumerate(alphabet):
        table[ord(c)] = table[ord(c.lower())] = i
    return lambda raw: table[raw]


def _make(route, pattern, literal, span, shift, rng, lens_by_off=None):
    enc, alphabet, letters, codes = ROUTES[route]
    lens_by_off = lens_by_off or edge_lengths(span)
    rows, offs = [], []
    for off, lens in lens_by_off:
        for n in lens:
            rows.append(_row(n, pattern, literal, rng, letters))
            offs.append(off)
    poison = _instance(pattern, literal, rng, _pattern_letters(route)).encode()
    view = View(rows, offs, poison, shift, _codes_of(alphabet) if codes else None)
    return view, (enc if codes else BaseEncoding), enc, alphabet


def _check(matcher, view, arr_enc, alphabet, pattern, literal, mode):
    seq = view.array(arr_enc)
    want = mo.matches(view.rows, pattern, mode, literal, alphabet)
    lazy = matcher.rolling_window(seq, mode=mode)
    n_want = np.array([sum(r) for r in want], dtype=np.int64)
    assert lazy.sum(axis=-1).cpu().numpy().tolist() == n_want.tolist()
    assert not lazy.is_materialised()
    got = lazy.tolist()
    assert got == want
    assert lazy.sum(axis=-1).cpu().numpy().tolist() == n_want.tolist()          # materialised path
    return lazy


def _matcher(kind, pattern, enc, route):
    if kind == "literal":
        return StringMatcher(pattern, enc)
    if kind == "gaps":
        return RegexMatcher(pattern, enc)
    return FixedLenRegexMatcher(pattern, enc)


@gpu
@pytest.mark.parametrize("route", list(ROUTES))
@pytest.mark.parametrize("m", LENS)
def test_rows_at_segment_edges(route, m):
    rng = random.Random(m * 100 + len(route))
    for kind, pattern, literal in _patterns(route, m):
        matcher = _matcher(kind, pattern, ROUTES[route][0], route)
        view, arr_enc, enc, alphabet = _make(route, pattern, literal, m, shift=(m + len(kind)) % 16, rng=rng)
        _check(matcher, view, arr_enc, alphabet, pattern, literal, "valid")
        _check(matcher, view, arr_enc, alphabet, pattern, literal, "same")


@gpu
@pytest.mark.parametrize("route", list(ROUTES))
@pytest.mark.parametrize("pattern", ["A.{0,3}C", "A.{,1}[CG]", "AC.{1,2}A.{0,2}C", "[AC].{2,5}[AC]C", "..", "A"])
def test_gaps_and_all_dot_patterns(route, pattern):
    rng = random.Random(len(pattern) + len(route))
    kind = "gaps" if "{" in pattern else "class"
    span = mo.span(pattern)
    matcher = _matcher(kind, pattern, ROUTES[route][0], route)
    for shift in (0, 5, 15):
        view, arr_enc, enc, alphabet = _make(route, pattern, False, span, shift, rng)
        _check(matcher, view, arr_enc, alphabet, pattern, False, "same")
        _check(matcher, view, arr_enc, alphabet, pattern, False, "valid")


@gpu
def test_reference_goldens_on_the_gpu():
    assert bnp.match_string(["ACGT", "TACTAC"], "AC").tolist() == [[T, F, F], [F, T, F, F, T]]
    seqs = bnp.as_encoded_array(["V1-1", "V2-1", "V1-1*2"])
    assert StringMatcher("V1-1", BaseEncoding).rolling_window(seqs).tolist() == [[T], [F], [T, F, F]]
    dna = bnp.as_encoded_array(["ACGT", "AATGAT"], bnp.DNAEncoding)
    assert FixedLenRegexMatcher("[AG].[AT]", bnp.DNAEncoding).rolling_window(dna).tolist() == \
        mo.matches([b"ACGT", b"AATGAT"], "[AG].[AT]", alphabet="ACGT")
    dna = bnp.as_encoded_array(["ACGTTCG", "AATGAAAC"], bnp.DNAEncoding)
    assert RegexMatcher("AA.{,1}[CT]", bnp.DNAEncoding).rolling_window(dna).tolist() == \
        [[F] * 7, [T, F, F, F, T, T, F, F]]
    acgt = bnp.as_encoded_array(["ACA", "TACTAC"], bnp.AlphabetEncoding("ACGT"))
    assert bnp.match_string(acgt, "AC").tolist() == [[T, F], [F, T, F, F, T]]
    aa = bnp.as_encoded_array(["AAACCC", "EEAAF"], bnp.AminoAcidEncoding)
    assert RegexMatcher("AA", bnp.AminoAcidEncoding).rolling_window(aa, mode="same").tolist() == \
        [[T, T, F, F, F, F], [F, F, T, F, F]]
    tutorial = ["CGTTAATTAC", "TCCTCCGGAAT", "TTGTCCTACACT", "ACCTAGCATACCC", "ATGTAGCGTCGACT", "CGCACGCTCGTTCAG",
                "GTCCACGTTAGTCCTG", "GGGTTAAGTAGTTTAGT", "CACAATGTTTCCGCTATG", "CGCTTCCAGGTTTTTAACC"]
    assert np.sum(bnp.match_string(bnp.as_encoded_array(tutorial), "AC"), axis=1).cpu().tolist() == \
        [1, 0, 2, 2, 1, 1, 1, 0, 1, 1]
    flat = bnp.match_string(bnp.as_encoded_array("TACTAC"), "AC")
    assert flat.cpu().tolist() == [F, T, F, F, T]
    windows = EncodedArray(torch.tensor([[0, 1], [1, 0], [0, 1]], dtype=torch.uint8, device="cuda"), bnp.DNAEncoding)
    assert StringMatcher("AC", bnp.DNAEncoding)(windows).cpu().tolist() == [T, F, T]
    assert FixedLenRegexMatcher("[AC]A", bnp.DNAEncoding)(windows).cpu().tolist() == [F, T, F]


@gpu
def test_raw_text_is_exact_and_encoded_text_is_case_folded():
    seqs = ["acACNn.A", "NNAC."]
    assert bnp.match_string(seqs, "AC").tolist() == mo.matches([s.encode() for s in seqs], "AC", literal=True)
    assert bnp.match_string(seqs, "N.").tolist() == [[F, F, F, F, F, F, F], [F, F, F, F]]
    assert FixedLenRegexMatcher("N.", BaseEncoding).rolling_window(seqs).tolist() == \
        mo.matches([s.encode() for s in seqs], "N.")
    dna = ["acgtACGT", "ttac"]
    assert StringMatcher("ac", bnp.DNAEncoding).rolling_window(dna).tolist() == \
        mo.matches([s.encode() for s in dna], "AC", literal=True, alphabet="ACGT")


@gpu
def test_fused_reductions_equal_the_materialised_result():
    rng = random.Random(3)
    rows = ["".join(rng.choice("ACGT") for _ in range(rng.randint(0, 300))) for _ in range(500)] + ["", "A", "AC"]
    seq = bnp.as_encoded_array(rows)
    for matcher, pattern, mode, alphabet in ((StringMatcher("ACT", bnp.DNAEncoding), "ACT", "valid", "ACGT"),
                                             (RegexMatcher("A.{0,2}C", bnp.DNAEncoding), "A.{0,2}C", "same", "ACGT"),
                                             (StringMatcher("ACT", BaseEncoding), "ACT", "valid", None)):
        lazy = matcher.rolling_window(seq, mode=mode)
        s, a, mean = lazy.sum(axis=-1), lazy.any(axis=-1), lazy.mean(axis=-1)
        assert not lazy.is_materialised()
        want = mo.counts([r.encode() for r in rows], pattern, mode, alphabet=alphabet)
        assert s.cpu().numpy().tolist() == want.tolist()
        lazy.ravel()
        assert lazy.is_materialised()
        assert torch.equal(lazy.sum(axis=-1), s) and torch.equal(lazy.any(axis=-1), a)
        assert torch.allclose(lazy.mean(axis=-1), mean, equal_nan=True)
        n = lazy.lengths.cpu().numpy()
        assert np.isnan(mean.cpu().numpy()[n == 0]).all()
        assert a.dtype == torch.bool and mean.dtype == torch.float64


@gpu
def test_fused_count_runs_only_the_count_kernel(big_fq_path, monkeypatch):
    """The fused sum calls the count entry point once and nothing else of the library, allocates no boolean output and
    leaves the result unmaterialised.  The profiler can drop kernel records, so it only has to agree where it has any:
    every match kernel it saw is a count build."""
    seq = bnp.open(big_fq_path).read().sequence
    real = ops.lib()

    class Calls:
        names = []

        def __getattr__(self, name):
            self.names.append(name)
            return getattr(real, name)

    calls = Calls()
    monkeypatch.setattr(ops, "lib", lambda: calls)
    for matcher in (StringMatcher("ACT", bnp.DNAEncoding), StringMatcher("ACT", BaseEncoding)):
        lazy = matcher.rolling_window(seq)
        torch.cuda.synchronize()
        before = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        calls.names.clear()
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            counts = lazy.sum(axis=-1)
            torch.cuda.synchronize()
        assert calls.names == ["bnpk_rows_match_count"], calls.names
        names = [e.name for e in prof.events() if "bnpk::rows_match" in e.name]
        assert all("rows_match_kernel<9" in n or "rows_match_generic_kernel<false" in n for n in names), set(names)
        assert torch.cuda.max_memory_allocated() - before < int(lazy.lengths.sum()) // 4
        assert not lazy.is_materialised()
        lazy.ravel()
        assert lazy.is_materialised() and torch.equal(counts, lazy.sum(axis=-1))


@gpu
@pytest.mark.parametrize("route", ["raw", "acgt_text", "acgtn"])
@pytest.mark.parametrize("pattern", ["ACGTTGCA", "A.{0,3}C.{1,2}G", "[AC]" + "G" * 30 + "[AT]"])
def test_long_rows_cut_into_pieces(route, pattern):
    """Rows longer than 2^14 positions are cut into pieces; matches straddling piece borders count once, and in
    "same" mode the row's last span - 1 positions are tested once, by its last piece."""
    rng = random.Random(len(pattern))
    enc, alphabet, letters, _ = ROUTES[route]
    span = mo.span(pattern)
    rows = []
    for n in (16384 + span - 1, 16384 + span, 40000, 70001, 5):
        r = bytearray(_row(n, pattern, False, rng, "ACGT"))
        for border in range(16384, n, 16384):
            for d in (-span, -span // 2, -1, 0):
                inst = _instance(pattern, False, rng, "ACGT").encode()
                p = border + d
                if 0 <= p and p + len(inst) <= n:
                    r[p:p + len(inst)] = inst
        tail = _instance(pattern, False, rng, "ACGT").encode()
        if len(tail) <= n:
            r[n - len(tail):] = tail
        rows.append(bytes(r))
    seq = bnp.as_encoded_array([r.decode() for r in rows])
    kind = "gaps" if "{" in pattern else "class"
    matcher = _matcher(kind, pattern, enc, route)
    for mode in ("same", "valid"):
        want = mo.matches(rows, pattern, mode, False, alphabet)
        got = matcher.rolling_window(seq, mode=mode)
        counts = got.sum(axis=-1).cpu().numpy().tolist()
        assert counts == [sum(w) for w in want]
        assert got.tolist() == want


@gpu
@pytest.mark.parametrize("route", ["acgt_text", "lut_tgca", "acgtn", "amino_text"])
def test_bad_bytes_raise_the_oracles_offset(route):
    enc, alphabet, letters, _ = ROUTES[route]
    rng = random.Random(5)
    span = 5
    pattern = _pattern_letters(route)[:2] * 2 + _pattern_letters(route)[0]
    bad_byte = b"#"
    places = [0, 7, 2047, 2048 - span, 1030, 3000]
    for n, pos in [(4000, p) for p in places] + [(40000, 20000), (40000, 16384 + 2), (4000, 3999)]:
        rows = [_row(300, pattern, True, rng, letters), _row(n, pattern, True, rng, letters)]
        rows[1] = rows[1][:pos] + bad_byte + rows[1][pos + 1:]
        with pytest.raises(mo.OracleEncodingError) as want:
            mo.matches(rows, pattern, alphabet=alphabet, literal=True)
        seq = bnp.as_encoded_array([r.decode() for r in rows])
        for reduce in (False, True):
            with pytest.raises(EncodingError) as got:
                res = StringMatcher(pattern, enc).rolling_window(seq)
                res.sum(axis=-1) if reduce else res.ravel()
            assert got.value.offset == want.value.offset, (n, pos, reduce)


@gpu
def test_reads_of_big_fq_and_selecting_entries(big_fq_path):
    """The reference's subsample example: keep the reads that contain "ACT"."""
    chunks = list(bnp.open(big_fq_path).read_chunks(50000))
    assert len(chunks) > 1
    for chunk in chunks:
        seq = chunk.sequence
        rows = [bytes(r) for r in o_rows(seq)]
        want = mo.counts(rows, "ACT", literal=True)
        counts = np.sum(bnp.match_string(seq, "ACT"), axis=1)
        assert counts.cpu().numpy().tolist() == want.tolist()
        kept = chunk[counts > 0]
        assert len(kept) == int((want > 0).sum())
        assert [bytes(r) for r in o_rows(kept.sequence)] == [r for r, c in zip(rows, want) if c > 0]
        assert kept.name.tolist() == [n for n, c in zip(chunk.name.tolist(), want) if c > 0]
        dna = StringMatcher("ACT", bnp.DNAEncoding).rolling_window(seq).sum(axis=-1)
        assert dna.cpu().numpy().tolist() == mo.counts(rows, "ACT", literal=True, alphabet="ACGT").tolist()


def o_rows(seq):
    flat = seq.ravel().raw().cpu().numpy().tobytes()
    out, p = [], 0
    for n in seq.lengths.cpu().numpy().tolist():
        out.append(flat[p:p + n])
        p += n
    return out


@gpu
def test_sacCer3_whole_genome(tmp_path):
    raw = gzip.open(os.path.join(GOLDEN, "sacCer3.fa.gz")).read()
    path = tmp_path / "sacCer3.fa"
    path.write_bytes(raw)
    whole = np.frombuffer((raw if raw.endswith(b"\n") else raw + b"\n") + b">", dtype=np.uint8)
    _, _, _, flat, seq_lens = o.multiline_fasta_split(whole)
    flat = np.asarray(flat, dtype=np.uint8).tobytes()
    rows, p = [], 0
    for n in seq_lens:
        rows.append(flat[p:p + n])
        p += n
    seq = bnp.open(str(path)).read().sequence
    assert len(seq) == 17
    cg = bnp.match_string(seq, "CG")
    assert cg.sum(axis=-1).cpu().numpy().tolist() == mo.counts(rows, "CG", literal=True).tolist()
    gapped = RegexMatcher("CG.{2,4}[AT]A", BaseEncoding).rolling_window(seq)
    assert gapped.sum(axis=-1).cpu().numpy().tolist() == mo.counts(rows, "CG.{2,4}[AT]A", "same").tolist()
    dna = StringMatcher("CG", bnp.DNAEncoding).rolling_window(seq)
    assert dna.mean(axis=-1).cpu().numpy().tolist() == \
        [c / max(len(r) - 1, 0) for c, r in zip(mo.counts(rows, "CG", literal=True, alphabet="ACGT"), rows)]


@gpu
def test_two_streams_and_the_dispatcher_op():
    from bionumpy_b200 import torch_ops
    top = torch_ops.load()
    rng = random.Random(11)
    jobs = []
    for route, pattern in (("lut_tgca", "AC.G"), ("amino_text", "[AC]DE")):
        span = mo.span(pattern)
        view, arr_enc, enc, alphabet = _make(route, pattern, False, span, 3, rng)
        jobs.append((view, enc, alphabet, pattern, FixedLenRegexMatcher(pattern, enc)._pattern))
    streams = [torch.cuda.Stream(), torch.cuda.Stream()]
    outs = []
    for (view, enc, alphabet, pattern, pat), s in zip(jobs, streams):
        with torch.cuda.stream(s):
            rows = pat.rows(view.array(BaseEncoding))
            args = (rows.enc_mode, pat.alphabet_size, pat.sets(view.base.device), pat.sub_lens)
            outs.append((rows, args) + ops.rows_match(view.base, view.starts, view.lens, *args, lut=rows.lut)[:2])
    torch.cuda.synchronize()
    for (view, enc, alphabet, pattern, pat), (rows, args, got, offsets) in zip(jobs, outs):
        want = mo.matches(view.rows, pattern, "valid", False, alphabet)
        assert got.cpu().numpy().astype(bool).tolist() == [x for r in want for x in r]
        mode, a_size, sets, sub_lens = args
        t, status = top.rows_match(view.base, view.starts, view.lens, mode, rows.lut, a_size, sets, sub_lens, False,
                                   offsets, int(offsets[-1]))
        assert torch.equal(t, got)
