"""The genome-side input path against the oracle, bit for bit: the multi-line FASTA buffer and reader
(multiline_flags_kernel, multiline_entries_kernel, io/multiline.py), indexed FASTA (interval_check_kernel,
interval_copy_kernel, io/indexed_fasta.py), the Bloom filter (bloom_insert_kernel, bloom_query_kernel), KmerIndex /
KmerLookup, the byte count (count_byte_kernel) and the per-row bincount (bincount_rows_kernel).

Every case that has to reach a second grid-stride pass sizes itself from bnpk_sm_count() and the launch shape the
kernel's entry point uses (csrc/misc_kernels.cu; csrc/interval_kernels.cu for the indexed FASTA gather), so the cases
stay meaningful on any SM count."""
import numpy as np
import pytest
import torch

from oracle import bnp_oracle as oracle

pytestmark = pytest.mark.gpu

# launch shapes of csrc/misc_kernels.cu and csrc/interval_kernels.cu: blocks per SM x threads per block (x work per thread)
THREADS = 256
LINE_BLOCKS_PER_SM = 8          # bnpk_multiline_flags / bnpk_multiline_entries: one line per thread
WARP_ROW_BLOCKS_PER_SM = 8      # bnpk_bincount_rows: one row per warp
COPY_BLOCKS_PER_SM = 8          # bnpk_interval_gather, copy pass: one row per COPY_LANES_PER_ROW threads
COPY_LANES_PER_ROW = 8
BLOOM_BLOCKS_PER_SM = 16        # bnpk_bloom_insert / bnpk_bloom_query: one value per thread
COUNT_BYTE_BLOCKS_PER_SM = 8    # bnpk_count_byte: one 16-byte unit per thread
POISON = np.frombuffer(b">\r\n", dtype=np.uint8)


@pytest.fixture(scope="module")
def bnp():
    import bionumpy_b200 as bnp
    return bnp


@pytest.fixture(scope="module")
def sm_count(bnp):
    from bionumpy_b200 import _native as nv
    return int(nv.lib().bnpk_sm_count())


def _flat(r):
    """Flat bytes (numpy) and row lengths of an (Encoded)RaggedArray."""
    return r.ravel().raw().cpu().numpy(), r._lens.cpu().numpy().astype(np.int64)


def _rows_bytes(r):
    flat, lens = _flat(r)
    ends = np.cumsum(lens)
    return [flat[e - n:e].tobytes() for e, n in zip(ends, lens)]


def _b(text):
    return np.frombuffer(text, dtype=np.uint8)


def _letters(rng, n, alphabet=b"ACGTacgtN"):
    return rng.choice(_b(alphabet), size=n).tobytes()


def _device_view(host, offset):
    """``host`` on the device as a view at byte ``offset`` of a larger allocation, every other byte poison."""
    n = host.size
    total = offset + n + 32
    base = np.resize(POISON, total).copy()
    base[offset:offset + n] = host
    dev = torch.from_numpy(base).cuda()
    assert dev.data_ptr() % 16 == 0
    return dev[offset:offset + n]


# ------------------------------------------------------------------------------------------------------------------
# 1. multi-line FASTA, buffer level
# ------------------------------------------------------------------------------------------------------------------
def _lines_text(lines, eol=b"\n"):
    return b"".join(l + eol for l in lines)


def _mixed_width_entry(rng):
    widths = [1, 2, 59, 60, 61, 4097, 60, 1, 61, 2, 59]
    return [b">mixed widths"] + [_letters(rng, w) for w in widths]


def _multiline_cases():
    rng = np.random.default_rng(41)
    cases = {}
    cases["blank_lines"] = b">a x\nACGT\n\nGG\n\n\n>b\n\nTT\n\n>c\nA\n>"
    cases["header_only_middle"] = b">a\nAC\n>b only\n>c desc\nGT\nT\n>d\n>e\n>"
    cases["bare_header"] = b">\nACG\n>\n>x\nA\n>\n\n>"
    cases["gt_inside_line"] = b">a\nAC>GT\nT>\n>>b\nA>>\n>c\n>G\n>"
    cases["mixed_widths"] = _lines_text(_mixed_width_entry(rng) + [b">second", _letters(rng, 60), _letters(rng, 4097)]) + b">"
    cases["one_long_line"] = _lines_text([b">long", _letters(rng, 3 * 2048 + 123), b">short", b"ACG"]) + b">"
    cases["all_crlf"] = _lines_text([b">a one", _letters(rng, 60), _letters(rng, 17), b">b", b"", _letters(rng, 5), b">c"],
                                    b"\r\n") + b">"
    lines = [b">first"] + [_letters(rng, 7) for _ in range(12)] + [b">second"] + [_letters(rng, 3) for _ in range(4)]
    cases["first_cr_on_line_9"] = b"".join(l + (b"\r\n" if i >= 9 else b"\n") for i, l in enumerate(lines)) + b">"
    cases["cr_from_line_10"] = b"".join(l + (b"\r\n" if i >= 10 else b"\n") for i, l in enumerate(lines)) + b">"
    cases["cr_only_in_tail"] = b">a\nAC\nGT\n>b\r\nAC\r\nG"
    cases["incomplete_tail"] = _lines_text([b">a", _letters(rng, 80), b">b", _letters(rng, 80)]) + b">c\nACGT\nAC"
    cases["cr_line_9_lines_after_10"] = b"".join(
        l + (b"\r\n" if i in (9, 11, 14) else b"\n") for i, l in enumerate(lines)) + b">"
    return cases


MULTILINE_CASES = _multiline_cases()


def _check_multiline_buffer(buf, host):
    size, h_starts, h_lens, flat, seq_lens = oracle.multiline_fasta_split(host)
    data = host[:size]
    assert buf.size == size
    assert buf.count_entries() == len(h_starts) == len(seq_lens)
    assert buf.n_lines == int(np.count_nonzero(data == 10)) - 1
    names = buf.get_field_by_number(0)
    seqs = buf.get_field_by_number(1)
    got_names, got_name_lens = _flat(names)
    assert np.array_equal(got_name_lens, h_lens)
    assert np.array_equal(got_names, oracle.gather_rows(data, h_starts, h_lens))
    got_seqs, got_seq_lens = _flat(seqs)
    assert np.array_equal(got_seq_lens, seq_lens)
    assert np.array_equal(got_seqs, flat)
    return h_lens.size


@pytest.mark.parametrize("case", sorted(MULTILINE_CASES))
def test_multiline_buffer_edges_vs_oracle(bnp, case):
    """from_raw_buffer on views at byte offsets 0..15: size, entry count, line count, every name and sequence."""
    from bionumpy_b200.io.multiline import CudaMultiLineFastaBuffer
    host = _b(MULTILINE_CASES[case])
    for offset in range(16):
        buf = CudaMultiLineFastaBuffer.from_raw_buffer(_device_view(host, offset))
        _check_multiline_buffer(buf, host)


def test_multiline_buffer_cr_trimming_pinned(bnp):
    """The '\\r' probe looks at the first ten lines of the chunk: a '\\r' first seen on line 9 trims every line, one
    first seen on line 10 stays in the sequence."""
    from bionumpy_b200.io.multiline import CudaMultiLineFastaBuffer
    for case, trimmed in (("first_cr_on_line_9", True), ("cr_from_line_10", False)):
        host = _b(MULTILINE_CASES[case])
        seqs = CudaMultiLineFastaBuffer.from_raw_buffer(_device_view(host, 5)).get_field_by_number(1)
        flat, _ = _flat(seqs)
        assert (13 in flat.tolist()) != trimmed, case


@pytest.mark.parametrize("text", [b">a\nACGT\nGG", b">a\nACGT\n", b">only a header", b">a\nA>\n", b">a\nAC\nGT\n\n"])
def test_multiline_buffer_without_complete_entry(bnp, text):
    from bionumpy_b200.io.exceptions import IncompleteEntryException
    from bionumpy_b200.io.multiline import CudaMultiLineFastaBuffer
    host = _b(text)
    with pytest.raises(oracle.OracleIncompleteEntry):
        oracle.multiline_fasta_split(host)
    for offset in (0, 7):
        with pytest.raises(IncompleteEntryException):
            CudaMultiLineFastaBuffer.from_raw_buffer(_device_view(host, offset))


@pytest.mark.parametrize("shape", ["short_lines", "many_entries"])
def test_multiline_buffer_second_grid_stride_pass(bnp, sm_count, shape):
    """More lines than one grid of the flags and entries kernels covers: both take a second grid-stride pass."""
    from bionumpy_b200.io.multiline import CudaMultiLineFastaBuffer
    one_pass = sm_count * LINE_BLOCKS_PER_SM * THREADS
    n_lines = one_pass + 1000
    rng = np.random.default_rng(7)
    letters = [bytes([c]) for c in rng.choice(_b(b"ACGTacgtN"), size=n_lines)]
    if shape == "short_lines":
        # three entries of width-1 lines (some blank), the last two headers after the first grid
        half = n_lines // 2
        lines = [b">a"] + [c if w else b"" for c, w in zip(letters[:half], rng.integers(0, 2, size=half))]
        lines += [b">b"] + letters[half:] + [b">c", b"A"]
    else:
        # entries of a bare or named header and 0..2 one-byte lines: an entry starts every one to three lines
        lines = []
        for c, r, n_seq in zip(letters, rng.random(n_lines), rng.integers(0, 3, size=n_lines)):
            lines.append(b">" if r < 0.5 else b">e")
            lines += [c] * int(n_seq)
            if len(lines) >= n_lines:
                break
    host = _b(_lines_text(lines) + b">")
    assert host.size < (1 << 20) and np.count_nonzero(host == 10) > one_pass
    for offset in (0, 3):
        buf = CudaMultiLineFastaBuffer.from_raw_buffer(_device_view(host, offset))
        n_entries = _check_multiline_buffer(buf, host)
        assert buf.n_lines > one_pass
        assert n_entries == (3 if shape == "short_lines" else int(np.count_nonzero(host == ord(">"))) - 1)


# ------------------------------------------------------------------------------------------------------------------
# 2. multi-line FASTA, reader level
# ------------------------------------------------------------------------------------------------------------------
def _oracle_whole_file(raw):
    whole = _b((raw if raw.endswith(b"\n") else raw + b"\n") + b">")
    size, h_starts, h_lens, flat, seq_lens = oracle.multiline_fasta_split(whole)
    names = [whole[s:s + n].tobytes() for s, n in zip(h_starts, h_lens)]
    ends = np.cumsum(seq_lens)
    return names, [flat[e - n:e].tobytes() for e, n in zip(ends, seq_lens)]


def _read_chunked(bnp, path, min_chunk_size):
    names, seqs = [], []
    for chunk in bnp.open(str(path)).read_chunks(min_chunk_size=min_chunk_size):
        names += _rows_bytes(chunk.name)
        seqs += _rows_bytes(chunk.sequence)
    return names, seqs


def _small_fasta(eol=b"\n"):
    rng = np.random.default_rng(3)
    lines = [b">a first", _letters(rng, 9), _letters(rng, 9), _letters(rng, 4), b">b", b">c", _letters(rng, 1), b"",
             _letters(rng, 12), b">", _letters(rng, 5), b">d tail", _letters(rng, 9), _letters(rng, 2)]
    return eol.join(lines)


SMALL_FILES = {
    "final_newline": _small_fasta() + b"\n",
    "no_final_newline": _small_fasta(),
    "ends_in_blank_line": _small_fasta() + b"\n\n",
    "header_only_last": _small_fasta() + b"\n>last\n",
    "header_only_last_no_newline": _small_fasta() + b"\n>last",
    "crlf": _small_fasta(b"\r\n") + b"\r\n",
}


@pytest.mark.parametrize("name", sorted(SMALL_FILES))
def test_multiline_reader_every_cut_vs_oracle(bnp, tmp_path, name):
    """bnp.open(...).read_chunks(min_chunk_size) for every chunk size up to the file's length (so every first cut
    position) equals the oracle's split of the whole file with '\\n>' appended."""
    raw = SMALL_FILES[name]
    path = tmp_path / "small.fa"
    path.write_bytes(raw)
    want = _oracle_whole_file(raw)
    if name.startswith("header_only_last"):
        assert want[0][-1] == b"last" and want[1][-1] == b""
    assert _read_chunked(bnp, path, 1 << 20) == want
    for size in range(1, len(raw) + 2):
        assert _read_chunked(bnp, path, size) == want, size
    data = bnp.open(str(path)).read()
    assert (_rows_bytes(data.name), _rows_bytes(data.sequence)) == want


def test_multiline_reader_entries_larger_than_the_chunk(bnp, tmp_path):
    """Entries far larger than the chunk size: the reader grows the buffer until an entry completes."""
    rng = np.random.default_rng(8)
    parts = []
    for i, (L, w) in enumerate([(3000, 60), (0, 60), (12345, 80), (1, 7), (70000, 4097), (500, 1)]):
        seq = _letters(rng, L)
        parts.append(b">c%d desc\n" % i + b"".join(seq[a:a + w] + b"\n" for a in range(0, L, w)))
    raw = b"".join(parts)
    path = tmp_path / "big.fa"
    path.write_bytes(raw)
    want = _oracle_whole_file(raw)
    for size in (5, 64, 1000, 4096, 50_000, 5_000_000):
        assert _read_chunked(bnp, path, size) == want, size


# ------------------------------------------------------------------------------------------------------------------
# 3. indexed FASTA
# ------------------------------------------------------------------------------------------------------------------
WIDTHS = (1, 7, 60, 80, 4096)


def _indexed_contigs(rng):
    """(name, sequence, line width): lengths 1, w - 1, w, w + 1 and 3w for every width, an empty contig in the
    middle and one contig of more than 1 MB."""
    contigs = []
    for w in WIDTHS:
        for L in sorted({1, w - 1, w, w + 1, 3 * w} - {0}):
            contigs.append((f"w{w}_L{L}", _letters(rng, L, b"ACGTNacgt"), w))
        if w == 60:
            contigs.append(("empty", b"", 60))
    contigs.append(("big", _letters(rng, 1_200_013, b"ACGT"), 80))
    contigs.append(("last", _letters(rng, 130, b"ACGT"), 60))
    return contigs


def _write_indexed(path, contigs, eol, trailing):
    out = []
    for name, seq, w in contigs:
        out.append(b">" + name.encode() + b" some description" + eol)
        out += [seq[a:a + w] + eol for a in range(0, len(seq), w)]
    raw = b"".join(out)
    if not trailing:
        raw = raw[:-len(eol)]
    path.write_bytes(raw)
    return _b(raw)


def _intervals(rng, contigs, n_min):
    iv = []
    for name, seq, w in contigs:
        L = len(seq)
        iv += [(name, 0, 0), (name, L, L), (name, 0, L)]
        if L == 0:
            continue
        iv.append((name, L - 1, L))
        if L <= 3 * 80 + 1:
            iv += [(name, i, i + 1) for i in range(L)]                 # every length-1 interval
            iv += [(name, i, i) for i in range(0, L, max(L // 5, 1))]  # empty ones inside
        if L <= 3 * 4096:
            for j in range(0, L + 1, w):                               # every line boundary of the contig
                iv += [(name, j, L), (name, 0, j), (name, j, min(j + w, L))]
                if 0 < j < L:
                    iv.append((name, j - 1, j + 1))
        else:
            iv += [(name, j - 1, j + 1) for j in range(w, L, 997 * w)]
        if L > 1_000_000:
            iv += [(name, 1, L - 1), (name, 12345, 12345 + (1 << 20) + 7)]
    while len(iv) < n_min:
        name, seq, w = contigs[int(rng.integers(len(contigs)))]
        a = int(rng.integers(0, len(seq) + 1))
        iv.append((name, a, int(rng.integers(a, min(len(seq), a + 300) + 1))))
    return iv


def _check_intervals(fa, data, idx, truth, iv):
    seqs = fa.get_interval_sequences(iv)
    flat, lens = _flat(seqs)
    assert np.array_equal(lens, [b - a for _, a, b in iv])
    pos = 0
    for c, a, b in iv:
        want = _b(truth[c][a:b]) if idx[c]["lenc"] == 0 else oracle.indexed_fasta_interval(data, idx[c], a, b)
        assert want.tobytes() == truth[c][a:b]
        assert flat[pos:pos + b - a].tobytes() == want.tobytes(), (c, a, b)
        pos += b - a


@pytest.mark.parametrize("trailing", [True, False], ids=["final_newline", "no_final_newline"])
@pytest.mark.parametrize("eol", [b"\n", b"\r\n"], ids=["lf", "crlf"])
def test_indexed_fasta_vs_oracle(bnp, sm_count, tmp_path, eol, trailing):
    """create_index and a .fai written from the oracle's index; whole contigs and intervals of every kind (empty, on
    every line boundary, every single base of the small contigs, the last base, more than 1 MB) in one call with more
    intervals than one grid of the gather kernel covers."""
    rng = np.random.default_rng(len(eol) * 2 + trailing)
    contigs = _indexed_contigs(rng)
    truth = {name: seq for name, seq, _ in contigs}
    path = tmp_path / "genome.fa"
    data = _write_indexed(path, contigs, eol, trailing)
    idx = oracle.fasta_index(data)
    from bionumpy_b200.io.indexed_fasta import create_index, read_index
    assert create_index(path) == idx
    assert [v["rlen"] for v in idx.values()] == [len(s) for _, s, _ in contigs]
    assert all(v["lenb"] - v["lenc"] == len(eol) for v in idx.values() if v["rlen"])
    one_pass = sm_count * COPY_BLOCKS_PER_SM * (THREADS // COPY_LANES_PER_ROW)
    iv = _intervals(rng, contigs, one_pass + 777)
    assert len(iv) > one_pass

    def check(fa):
        assert fa.get_contig_lengths() == {name: len(seq) for name, seq, _ in contigs}
        for name, seq, _ in contigs:
            assert fa[name].raw().cpu().numpy().tobytes() == seq, name
        _check_intervals(fa, data, idx, truth, iv)

    check(bnp.IndexedFasta(str(path)))
    fai = tmp_path / "genome.fa.fai"
    fai.write_text("".join(f"{n}\t{v['rlen']}\t{v['offset']}\t{v['lenc']}\t{v['lenb']}\n" for n, v in idx.items()))
    assert read_index(fai) == idx
    check(bnp.IndexedFasta(str(path)))


def test_indexed_fasta_interval_to_the_last_byte(bnp, tmp_path):
    """A file without a final newline: an interval that ends on the file's last byte works, one byte further is
    reported by the gather's check pass and raises; so does an interval that ends past its contig but inside the
    file, in the bytes of the next contig."""
    rng = np.random.default_rng(5)
    for L, w in ((120, 60), (121, 60), (5, 1), (4097, 4096)):
        contigs = [("a", _letters(rng, 33), 7), ("z", _letters(rng, L), w)]
        path = tmp_path / f"end_{L}_{w}.fa"
        data = _write_indexed(path, contigs, b"\n", trailing=False)
        fa = bnp.IndexedFasta(str(path))
        got = fa.get_interval_sequences([("z", L - 1, L), ("z", 0, L)])
        assert _rows_bytes(got) == [contigs[1][1][-1:], contigs[1][1]]
        assert data[-1] == contigs[1][1][-1]
        with pytest.raises(AssertionError, match="beyond the file"):
            fa.get_interval_sequences([("a", 0, 3), ("z", L - 1, L + 1)])
        with pytest.raises(AssertionError, match="beyond the file"):
            fa.get_interval_sequences([("z", 0, L + 1)])
        with pytest.raises(AssertionError, match="beyond the file"):
            fa.get_interval_sequences([("a", 0, 34)])


# ------------------------------------------------------------------------------------------------------------------
# 4. Bloom filter
# ------------------------------------------------------------------------------------------------------------------
MASK_SIZES = [1, 2, 3, 100003, 1 << 20, (1 << 27) + 1]


def _bloom_values(rng, n, negative):
    v = rng.integers(0, 1 << 62, size=n, dtype=np.int64, endpoint=True)
    v[: n // 8] = v[n // 8: n // 4]                                    # repeated values
    v[-5:] = [0, 1, (1 << 62), (1 << 40), 12345]
    if negative:
        v[n // 4: n // 2] = -v[n // 4: n // 2]
        v[n // 2: n // 2 + 7] = [-1, -2, -3, -7, -(1 << 62), np.iinfo(np.int64).min, -100003]
    return v


def _bloom_offsets(rng, n_hash, negative):
    off = rng.integers(0, 1 << 40, size=n_hash, dtype=np.int64, endpoint=True)
    off[0] = 1 << 40
    if negative:
        off[1::2] = -off[1::2] - 1
    return off


def _check_bloom(bnp, sm_count, mask_size, n_hash, negative):
    rng = np.random.default_rng(mask_size % 1000 + n_hash + 50 * negative)
    n = sm_count * BLOOM_BLOCKS_PER_SM * THREADS + 4321                  # more values than one grid covers
    values = _bloom_values(rng, n, negative)
    offsets = _bloom_offsets(rng, n_hash, negative)
    bf = bnp.BloomFilter(mask_size, offsets)
    bf.insert(torch.from_numpy(values[: n // 3]).cuda())               # two inserts accumulate
    bf.insert(values[n // 3:])
    mask = oracle.bloom_filter_mask(values, offsets, mask_size)
    assert np.array_equal(bf._mask.cpu().numpy().astype(bool), mask)
    probe = np.concatenate([values[::5], rng.integers(-(1 << 62), 1 << 62, size=n // 2, dtype=np.int64)])
    if not negative:
        probe = np.abs(probe)
    got = bf[torch.from_numpy(probe).cuda()].cpu().numpy()
    assert np.array_equal(got, oracle.bloom_filter_query(mask, probe, offsets))
    assert bool(bf[values].all().item())
    even = probe[: 2 * (probe.size // 2)]
    grid = bf[even.reshape(-1, 2)]
    assert grid.shape == (even.size // 2, 2) and np.array_equal(grid.cpu().numpy().ravel(), got[:even.size])
    # a sparse filter, where a value on the wrong slot changes the mask and the answers
    few = values[n // 4: n // 4 + max(1, min(mask_size // (4 * n_hash), 2000))]
    sparse = bnp.BloomFilter(mask_size, offsets)
    sparse.insert(few)
    mask = oracle.bloom_filter_mask(few, offsets, mask_size)
    assert np.array_equal(sparse._mask.cpu().numpy().astype(bool), mask)
    assert np.array_equal(sparse[probe].cpu().numpy(), oracle.bloom_filter_query(mask, probe, offsets))


@pytest.mark.parametrize("n_hash", [1, 3, 8])
@pytest.mark.parametrize("mask_size", MASK_SIZES)
def test_bloom_filter_vs_oracle(bnp, sm_count, mask_size, n_hash):
    """Values up to 2^62 and offsets up to 2^40, repeated values, more values than one grid covers."""
    _check_bloom(bnp, sm_count, mask_size, n_hash, negative=False)


@pytest.mark.parametrize("n_hash", [1, 3, 8])
@pytest.mark.parametrize("mask_size", MASK_SIZES)
def test_bloom_filter_negative_values_vs_oracle(bnp, sm_count, mask_size, n_hash):
    """Negative values and offsets: v ^ offset is reduced with NumPy's floor modulo, as the reference does."""
    _check_bloom(bnp, sm_count, mask_size, n_hash, negative=True)


def test_bloom_filter_floor_modulo_example(bnp):
    """offset 5, mask size 3: -1, -7 and -2^62 go to slots 0, 2 and 1 (NumPy's floor modulo of v ^ 5)."""
    values = np.array([-1, -7, -(1 << 62)], dtype=np.int64)
    assert ((values ^ 5) % 3).tolist() == [0, 2, 1]
    for v, slot in zip(values, (0, 2, 1)):
        bf = bnp.BloomFilter(3, [5])
        bf.insert(np.array([v]))
        assert bf._mask.cpu().tolist() == [int(j == slot) for j in range(3)]
        assert bf[values].cpu().tolist() == [s == slot for s in (0, 2, 1)]


@pytest.mark.parametrize("k", [5, 31])
def test_bloom_filter_from_hash_functions_and_sequences(bnp, k):
    rng = np.random.default_rng(k)
    lens = rng.integers(0, 90, size=300)
    flat = rng.integers(0, 4, size=int(lens.sum())).astype(np.uint8)
    ragged = bnp.EncodedRaggedArray(bnp.EncodedArray(torch.from_numpy(flat).cuda(), bnp.DNAEncoding), lens)
    kmers = bnp.get_kmers(ragged, k)
    h, _ = oracle.get_kmers(flat, lens, k)
    offsets = [0, 17, 1 << 40]
    bf = bnp.BloomFilter.from_hash_functions_and_seqeuences(offsets, kmers, 100003)
    mask = oracle.bloom_filter_mask(h, offsets, 100003)
    assert np.array_equal(bf._mask.cpu().numpy().astype(bool), mask)
    probe = rng.integers(0, 4 ** k, size=20000, dtype=np.int64)
    assert np.array_equal(bf[probe].cpu().numpy(), oracle.bloom_filter_query(mask, probe, offsets))


# ------------------------------------------------------------------------------------------------------------------
# 5. k-mer index
# ------------------------------------------------------------------------------------------------------------------
def _index_rows(rng, k, n_rows):
    rows = []
    for r in range(n_rows):
        kind = r % 7
        if kind == 0:
            rows.append(np.zeros(0, dtype=np.uint8))                                   # empty
        elif kind == 1:
            rows.append(rng.integers(0, 4, size=int(rng.integers(1, k + 1)) - 1).astype(np.uint8))  # shorter than k
        elif kind == 2:
            rows.append(np.full(k + int(rng.integers(0, 40)), r % 4, dtype=np.uint8))  # one k-mer repeated
        elif kind == 3:
            rows.append(np.tile(np.array([0, 1, 2], dtype=np.uint8), k + 5))           # a period-3 row, in many rows
        else:
            rows.append(rng.integers(0, 4, size=int(rng.integers(k, k + 80))).astype(np.uint8))
    lens = np.array([r.size for r in rows], dtype=np.int64)
    return np.concatenate(rows), lens


@pytest.mark.parametrize("k", [1, 5, 16, 31])
def test_kmer_index_vs_oracle(bnp, k):
    """Every key and its rows; both construction branches (chosen by h.max() and the row count, asserted here);
    absent hashes and strings; KmerLookup.get_sequences."""
    rng = np.random.default_rng(200 + k)
    n_rows = 700
    flat, lens = _index_rows(rng, k, n_rows)
    ragged = bnp.EncodedRaggedArray(bnp.EncodedArray(torch.from_numpy(flat).cuda(), bnp.DNAEncoding), lens)
    h, hl = oracle.get_kmers(flat, lens, k)
    want = oracle.kmer_index(h, hl)
    large_key_branch = int(h.max()) >= (1 << 62) // n_rows
    assert large_key_branch == (k == 31)
    index = bnp.KmerIndex.create_index(ragged, k)
    keys = sorted(want)
    assert index._keys.cpu().tolist() == keys
    assert index._rows.cpu().tolist() == [r for key in keys for r in want[key]]
    assert index._first.cpu().tolist() == np.concatenate([[0], np.cumsum([len(want[key]) for key in keys])]).tolist()
    assert max(len(v) for v in want.values()) > 50                     # keys shared by many rows
    for key in keys[:: max(len(keys) // 300, 1)] + [int(h[0]), int(h[-1])]:
        assert index.get_indices(key).cpu().tolist() == want[key]
        assert index.get_indices(oracle.kmer_to_string(key, k)).cpu().tolist() == want[key]
    absent = [x for x in rng.integers(0, 4 ** k, size=200, dtype=np.int64).tolist() if x not in want][:20]
    absent += [-1, 4 ** k, (1 << 62) + 1, keys[0] - 1, keys[-1] + 1]
    absent = [x for x in absent if x not in want]
    for key in absent:
        assert index.get_indices(key).numel() == 0
        if 0 <= key < 4 ** k:
            assert index.get_indices(oracle.kmer_to_string(key, k)).numel() == 0
    row_bytes = [flat[e - n:e].tobytes() for e, n in zip(np.cumsum(lens), lens)]
    lookup = bnp.KmerLookup.from_sequences(ragged, k)
    for key in [keys[0], keys[-1], max(want, key=lambda x: len(want[x]))] + absent[:2]:
        got = lookup.get_sequences(key)
        assert _rows_bytes(got) == [row_bytes[r] for r in want.get(key, [])]


# ------------------------------------------------------------------------------------------------------------------
# 6. byte count and per-row bincount
# ------------------------------------------------------------------------------------------------------------------
def test_count_byte_every_value_length_and_offset(bnp):
    """count_byte for all 256 byte values on lengths 0..48 at view offsets 0..15: one call per case into its own
    output word, one synchronisation at the end."""
    from bionumpy_b200 import _native as nv
    lib = nv.lib()
    rng = np.random.default_rng(13)
    span = 64
    host = np.empty((256, span), dtype=np.uint8)
    for v in range(256):
        # v at random positions, every other byte a near miss (one bit or one step away) or random
        near = np.array([v ^ (1 << rng.integers(8)) for _ in range(span)] + list((v + np.array([1, 255])) % 256))
        host[v] = np.where(rng.random(span) < 0.45, v, rng.choice(np.concatenate([near, rng.integers(0, 256, 8)]), span))
    base = torch.from_numpy(host.reshape(-1)).cuda()
    assert base.data_ptr() % 16 == 0
    out = torch.full((256, 16, 49), -1, dtype=torch.int64, device="cuda")
    s = nv.stream_ptr()
    b0, o0 = base.data_ptr(), out.data_ptr()
    for v in range(256):
        for off in range(16):
            for n in range(49):
                slot = ((v * 16) + off) * 49 + n
                nv.check(lib.bnpk_count_byte(b0 + v * span + off, n, v, o0 + 8 * slot, s))
    got = out.cpu().numpy()
    want = np.empty_like(got)
    for v in range(256):
        for off in range(16):
            want[v, off] = np.concatenate([[0], np.cumsum(host[v, off:off + 48] == v)])
    assert np.array_equal(got, want)


def test_count_byte_many_grid_passes(bnp, sm_count):
    """64 MiB + 7 bytes at offset 3: many grid-stride passes of the unaligned path plus the tail."""
    from bionumpy_b200 import ops
    n = (64 << 20) + 7
    assert n > sm_count * COUNT_BYTE_BLOCKS_PER_SM * THREADS * 16
    rng = np.random.default_rng(1)
    host = rng.integers(0, 256, size=n + 3, dtype=np.uint8)
    host[-1] = 10
    view = torch.from_numpy(host).cuda()[3:]
    for v in (10, 0, 255, ord("A")):
        assert ops.count_byte(view, v) == int(np.count_nonzero(host[3:] == v)), v
    aligned = torch.from_numpy(host[:n - 7].copy()).cuda()
    assert ops.count_byte(aligned, 10) == int(np.count_nonzero(host[:n - 7] == 10))


@pytest.mark.parametrize("n_bins", [1, 5, 16])
def test_bincount_rows_second_grid_pass(bnp, sm_count, n_bins):
    """More rows than one grid of the one-warp-per-row kernel covers, with empty rows and rows longer than a warp."""
    from bionumpy_b200 import ops
    n_rows = sm_count * WARP_ROW_BLOCKS_PER_SM * (THREADS // 32) * 2 + 333
    rng = np.random.default_rng(n_bins)
    lens = rng.integers(0, 12, size=n_rows)
    lens[rng.random(n_rows) < 0.3] = 0
    lens[-1] = 70
    values = rng.integers(0, n_bins * 3, size=int(lens.sum()), dtype=np.int64)
    offsets = torch.from_numpy(np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)).cuda()
    got, status = ops.bincount_rows(torch.from_numpy(values).cuda(), offsets, n_bins)
    assert ops.read_status(status).bad_base() is None
    assert np.array_equal(got.cpu().numpy(), oracle.count_rows(values % n_bins, lens, n_bins))
