"""The warp-specialised fused count splits the chunk into one contiguous tile range per CTA.  Every CTA but the first
guesses the line phase of its range's first byte from the bytes, stages its outputs range-locally and checks the guess
once, at the range's end (a wrong guess counts the range a second time, in the same launch).  These inputs put ragged
records, records longer than a tile, invalid records and long (deferred) rows at range starts; the histogram and the
status words must match the oracle, and every status word but the long-row count must match the register-staged
kernel, which resolves each tile's line index exactly."""
import numpy as np
import pytest
import torch

from helpers import make_fastq, oracle_hist
from oracle import bnp_oracle as o

pytestmark = pytest.mark.gpu

WS_REDO = 3          # workspace header word: ranges counted a second time (bnpk_device.cuh kWsRedo)


def same_words(st, ref):
    """Status words equal.  Which rows a kernel leaves to the long-row pass is its own choice: so N_LONG_ROWS is not
    compared, nor (when rows were left) the last row the kernel counted itself."""
    from bionumpy_b200 import _native as nv
    skip = {nv.ST_N_LONG_ROWS}
    if st.n_long_rows or ref.n_long_rows:
        skip |= {nv.ST_LAST_ROW_START, nv.ST_LAST_ROW_INDEX}
    return [w for i, w in enumerate(st.words) if i not in skip] == [w for i, w in enumerate(ref.words) if i not in skip]


@pytest.fixture(scope="module")
def ops():
    from bionumpy_b200 import ops
    return ops


def count(ops, chunk_np, k, bins, window=0, shift=0, **kw):
    """Fused count of chunk_np placed `shift` bytes into an aligned buffer (0: the warp-specialised kernel, 1: the
    register-staged one).  Returns (hist, status words, redo count)."""
    from bionumpy_b200 import _native as nv
    buf = torch.zeros(chunk_np.size + 32, dtype=torch.uint8, device="cuda")
    view = buf[shift: shift + chunk_np.size]
    view.copy_(torch.from_numpy(chunk_np).cuda())
    hist, status = ops.chunk_kmer_count(view, k, bins, window_size=window, **kw)
    ws = nv.workspace(chunk_np.size, view.device)
    redo = int(ws[8 * WS_REDO: 8 * WS_REDO + 8].view(torch.int64).item())
    return hist.cpu().numpy(), ops.read_status(status), redo


def check_against_references(ops, chunk, k=31, bins=1 << 14, window=0, redo=None):
    """Histogram and status words vs the oracle; every status word vs the register-staged kernel."""
    hist, st, n_redo = count(ops, chunk, k, bins, window)
    want, size, n_bases = oracle_hist(chunk, k, bins, window)
    _, starts, lens = o.fastq_split(chunk)
    assert (st.n_records, st.n_complete_bytes, st.n_bases) == (starts.shape[0], size, n_bases)
    assert st.n_values == want.sum() and not st.overflow
    assert st.bad_header_entry is None and st.bad_plus_entry is None and st.bad_base() is None
    assert np.array_equal(hist, want)
    ref_hist, ref_st, _ = count(ops, chunk, k, bins, window, shift=1)
    assert np.array_equal(ref_hist, want) and same_words(st, ref_st)
    if redo == 0:
        assert n_redo == 0
    elif redo == ">0":
        assert n_redo > 0
    return st


@pytest.mark.parametrize("window", [0, 41])
def test_ragged_fastq_guesses_every_phase(ops, window):
    """A few MB of ragged reads (quality lines start with '@' and '+' too): ~130 ranges, every guess right."""
    chunk = make_fastq(np.random.default_rng(40), 15000, 0, 300)
    assert chunk.size > 3_000_000
    check_against_references(ops, chunk, window=window, redo=0)
    if not window:
        check_against_references(ops, chunk, 7, 4 ** 7, redo=0)


def range_starts(n_bytes):
    """First byte of every CTA's range in a one-launch count of n_bytes (G = min(tiles, SMs) contiguous ranges)."""
    from bionumpy_b200 import _native as nv
    T = (n_bytes + 16383) // 16384
    G = min(T, nv.load_library().bnpk_sm_count())
    return np.array([c * T // G * 16384 for c in range(G)], dtype=np.int64)


def long_read_fastq(rng, n_records, length):
    """Records with `length`-base reads (numpy-built: Python strings of this size are slow)."""
    parts = []
    for r in range(n_records):
        seq = rng.choice(np.frombuffer(b"ACGT", dtype=np.uint8), size=length)
        qual = rng.integers(33, 74, size=length).astype(np.uint8)
        parts += [np.frombuffer(f"@long{r}\n".encode(), dtype=np.uint8), seq, np.frombuffer(b"\n+\n", dtype=np.uint8), qual,
                  np.frombuffer(b"\n", dtype=np.uint8)]
    return np.concatenate(parts)


@pytest.mark.parametrize("window", [0, 41])
def test_entries_longer_than_a_tile(ops, window):
    """12 kb reads: a header line and its sequence line fit in one tile only now and then, so some ranges find their
    phase in a later tile the ring holds and others are counted twice; the counts stay exact either way.  The sequence
    rows are longer than the row walk, so they go to the deferred list with their entry numbers."""
    chunk = make_fastq(np.random.default_rng(41), 300, 11000, 13000)
    st = check_against_references(ops, chunk, window=window)
    assert st.n_long_rows > 0


@pytest.mark.parametrize("window", [0, 41])
def test_second_pass_with_errors(ops, window):
    """150 kb reads: no window of the ring holds a header and its '+' line, so every range whose true phase is not 0
    is counted twice.  A bad header, a bad '+' line and a bad base, each inside such a range, are still reported with
    the oracle's entry numbers, and the counts stay exact."""
    chunk = long_read_fastq(np.random.default_rng(47), 60, 150_000)
    check_against_references(ops, chunk, window=window, redo=">0")
    starts_r = range_starts(chunk.size)
    nl = np.flatnonzero(chunk == 10)
    phase = np.searchsorted(nl, starts_r) % 4                  # line phase of every range's first byte
    bounds = np.append(starts_r, chunk.size)
    line_start = nl[:-1] + 1                                   # line i + 1 starts after newline i
    kind = (np.arange(1, nl.size)) % 4                         # 0 header, 1 sequence, 2 '+', 3 quality
    rng_of = np.searchsorted(bounds, line_start, side="right") - 1
    redone = (rng_of > 0) & (phase[np.clip(rng_of, 0, len(phase) - 1)] != 0)
    _, starts, lens = o.fastq_split(chunk)
    for k, name in ((0, "header"), (2, "plus"), (1, "base")):
        i = np.flatnonzero(redone & (kind == k))[0]
        entry = (i + 1) // 4
        bad = chunk.copy()
        bad[line_start[i] + (7 if k == 1 else 0)] = ord("N" if k == 1 else "#")
        hist, st, n_redo = count(ops, bad, 31, 1 << 14, window)
        ref_hist, ref_st, _ = count(ops, bad, 31, 1 << 14, window, shift=1)
        assert n_redo > 0 and same_words(st, ref_st), name
        if k == 1:
            assert st.bad_base() == (entry, 7)
        else:
            with pytest.raises(o.OracleFormatException) as e:
                o.fastq_split(bad)
            assert e.value.line_number // 4 == entry
            assert (st.bad_header_entry if k == 0 else st.bad_plus_entry) == entry, name
            assert np.array_equal(hist, ref_hist)


@pytest.mark.parametrize("window", [0, 41])
def test_long_rows_in_later_ranges(ops, window):
    """Rows over 1024 bases mixed with short ones in every range (deferred rows with global entry numbers)."""
    rng = np.random.default_rng(42 + window)
    parts = [make_fastq(rng, 1, 1100, 2500) if r % 7 == 0 else make_fastq(rng, 1, 45, 200) for r in range(12000)]
    chunk = np.concatenate(parts)
    check_against_references(ops, chunk, window=window)
    # a bad base deep inside a deferred row of a later range: reported by the long-row pass with the row's entry number
    _, starts, lens = o.fastq_split(chunk)
    entry = 10003 - 10003 % 7
    assert lens[entry, 1] > 1024
    chunk[starts[entry, 1] + 1030] = ord("N")
    _, st, _ = count(ops, chunk, 31, 1 << 14, window)
    assert st.bad_base() == (entry, 1030)


@pytest.mark.parametrize("window", [0, 41])
def test_errors_right_after_range_starts(ops, window):
    """The first header, the first '+' line and the first sequence row after the start of a range: the lines the
    range's phase is inferred from and the tile checks the F warp does itself."""
    base = make_fastq(np.random.default_rng(48), 15000, 60, 250)
    starts_e = _entry_offsets(base)[:-1]
    _, starts, lens = o.fastq_split(base)
    starts_r = range_starts(base.size)
    for c in (1, len(starts_r) // 2, len(starts_r) - 1):
        b = starts_r[c]
        for name in ("header", "plus", "base"):
            chunk = base.copy()
            if name == "header":
                entry = int(np.searchsorted(starts_e, b))
                chunk[starts_e[entry]] = ord("#")
            elif name == "plus":
                entry = int(np.searchsorted(starts[:, 2], b))
                chunk[starts[entry, 2]] = ord("-")
            else:
                entry = int(np.searchsorted(starts[:, 1], b))
                chunk[starts[entry, 1]] = ord("N")
            hist, st, n_redo = count(ops, chunk, 31, 1 << 14, window)
            ref_hist, ref_st, _ = count(ops, chunk, 31, 1 << 14, window, shift=1)
            assert n_redo == 0 and same_words(st, ref_st), (c, name)
            if name == "base":
                assert st.bad_base() == (entry, 0), c
            else:
                assert np.array_equal(hist, ref_hist), (c, name)
                with pytest.raises(o.OracleFormatException) as e:
                    o.fastq_split(chunk)
                assert e.value.line_number // 4 == entry
                assert (st.bad_header_entry if name == "header" else st.bad_plus_entry) == entry, (c, name)


def _entry_offsets(chunk):
    nl = np.flatnonzero(chunk == 10)
    return np.concatenate([[0], nl[3::4] + 1])            # first byte of every entry


@pytest.mark.parametrize("window", [0, 41])
def test_invalid_records_at_range_starts(ops, window):
    """A quality line that starts with '@' is valid; a bad header, a bad '+' line and a bad base deep inside the chunk
    (in later ranges, one each) must be reported with the oracle's entry numbers."""
    base = make_fastq(np.random.default_rng(43), 15000, 60, 250)
    starts_e = _entry_offsets(base)
    size, starts, lens = o.fastq_split(base)
    for kind, entry in (("header", 9000), ("plus", 11000), ("base", 12345), ("base", 7)):
        chunk = base.copy()
        if kind == "header":
            chunk[starts_e[entry]] = ord("#")
        elif kind == "plus":
            chunk[starts[entry, 2]] = ord("-")
        else:
            chunk[starts[entry, 1] + 5] = ord("N")
        hist, st, _ = count(ops, chunk, 31, 1 << 14, window)
        ref_hist, ref_st, _ = count(ops, chunk, 31, 1 << 14, window, shift=1)
        assert same_words(st, ref_st), kind
        if kind != "base":                                  # how a byte outside the alphabet is hashed is unspecified
            assert np.array_equal(hist, ref_hist), kind
        if kind == "base":
            assert st.bad_base() == (entry, 5)
            with pytest.raises(o.OracleEncodingError) as e:
                o.encode_flat(o.gather_rows(chunk, starts[:, 1], lens[:, 1]), o.alphabet_lut())
            assert e.value.offset == int(lens[:entry, 1].sum()) + 5
        else:
            with pytest.raises(o.OracleFormatException) as e:
                o.fastq_split(chunk)
            assert e.value.line_number // 4 == entry
            assert (st.bad_header_entry if kind == "header" else st.bad_plus_entry) == entry


def test_two_line_fasta(ops):
    rng = np.random.default_rng(44)
    parts = []
    for r in range(6000):
        L = int(rng.integers(0, 900)) if r % 40 else int(rng.integers(3000, 20000))
        parts.append(f">c{r} x\n{''.join(rng.choice(list('ACGT'), size=L)) if L else ''}\n")
    chunk = np.frombuffer("".join(parts).encode("ascii"), dtype=np.uint8).copy()
    size, starts, lens = o.two_line_fasta_split(chunk)
    codes = o.encode_flat(o.gather_rows(chunk, starts[:, 1], lens[:, 1]), o.alphabet_lut())
    for k, bins, window in ((21, 1 << 14, 0), (15, 1 << 12, 25)):
        vals, _ = o.get_minimizers_fast(codes, lens[:, 1], k, window) if window else o.get_kmers(codes, lens[:, 1], k)
        want = o.count_bucketed_flat(vals, bins)
        kw = dict(lines_per_entry=2, header_char=ord(">"), check_plus=False)
        hist, st, _ = count(ops, chunk, k, bins, window, **kw)
        ref_hist, ref_st, _ = count(ops, chunk, k, bins, window, shift=1, **kw)
        assert (st.n_records, st.n_complete_bytes, st.n_bases) == (6000, size, int(lens[:, 1].sum()))
        assert np.array_equal(hist, want) and np.array_equal(ref_hist, want)
        assert same_words(st, ref_st)


@pytest.mark.parametrize("window", [0, 41])
def test_sliced_launches_match_single(ops, window):
    """Slices of a ragged chunk (each launch its own ranges; the first range of a later slice starts from the carry)."""
    from bionumpy_b200 import _native as nv
    chunk_np = make_fastq(np.random.default_rng(45), 12000, 40, 400)
    whole, st_whole, _ = count(ops, chunk_np, 31, 1 << 14, window)
    chunk = torch.from_numpy(chunk_np).cuda()
    N = chunk.numel()
    for step in (1 << 20, 3 * 16384 + 100):
        hist = torch.zeros(1 << 14, dtype=torch.int64, device="cuda")
        status = nv.new_status(chunk.device)
        ws = nv.workspace(N, chunk.device)
        b = 0
        while b < N:
            e = min(N, b + step)
            nv.check(nv.lib().bnpk_chunk_kmer_count(nv.ptr(chunk), N, b, e, int(e == N), 4, ord("@"), 1, -1, 0, None, 31,
                                                    window, 1 << 14, 0, nv.ptr(hist), nv.ptr(status), nv.ptr(ws),
                                                    ws.numel(), nv.stream_ptr()))
            b = e
        assert np.array_equal(hist.cpu().numpy(), whole), step
        assert ops.read_status(status).words == st_whole.words, step


def test_host_pipeline_ragged(ops):
    chunk = make_fastq(np.random.default_rng(46), 15000, 0, 300)
    host = torch.from_numpy(chunk).pin_memory()
    want, size, n_bases = oracle_hist(chunk, 31, 1 << 14)
    _, starts, _ = o.fastq_split(chunk)
    pipe = ops.HostPipeline(host.numel(), slice_bytes=1 << 20)
    hist = torch.zeros(1 << 14, dtype=torch.int64, device="cuda")
    st = pipe.kmer_count(host, 31, hist)
    pipe.close()
    assert (st.n_records, st.n_complete_bytes, st.n_bases) == (starts.shape[0], size, n_bases)
    assert np.array_equal(hist.cpu().numpy(), want)
