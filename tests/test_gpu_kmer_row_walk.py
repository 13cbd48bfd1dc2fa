"""The k-mer build of the warp-specialised fused count (bnpk::ws::tile_ws_kernel) walks a 32-row chunk one lane per row,
block by block: as many blocks of 16 k-mers as the chunk's longest row has.  A row with fewer k-mers counts the rest
into a spare word, and every unit a row touches is validated once: whole where the walk encodes an interior unit,
masked at the row's first two units, its last unit and any unit past the walk.

These chunks put every k-mer count mod 16 at every row offset mod 16 (so rows end at every byte of a unit), mix rows of
10 and 11 units with rows that have no k-mer, hold 32-row chunks in which no row has one, and put bad bytes in units the
walk does not encode.  The histogram and all 16 status words are compared with the C oracle (oracle/kmer_oracle.c)."""
import numpy as np
import pytest
import torch

from oracle import bnp_oracle as o
from test_gpu_minimizer_count import Records
from test_oracle_goldens import c_oracle_hist

gpu = pytest.mark.gpu

K, BINS = 31, 1 << 14                     # the flagship shape: this table and k take the warp-specialised k-mer build
READ = 150                                # 120 k-mers: 10 units at row offsets 0..10 mod 16, 11 units at 11..15
LONG = 480                                # ends inside the 512-byte halo behind a tile: never left to the long-row pass
TILE = 16384
ENCODINGS = {"acgt": (0, "ACGT"), "actg": (1, "ACTG"), "lut_actg": (3, "ACTG")}


def expected_words(data, alphabet, bad=None):
    """The 16 status words of one count of `data`: complete FASTQ records, rows the row walk takes itself, no '\\r'.
    `bad`: the oracle's (row, position) of the first byte outside the alphabet."""
    from bionumpy_b200 import _native as nv
    r, _, stats = c_oracle_hist(data, K, BINS, alphabet=alphabet.encode())
    assert r >= 0
    _, starts, _ = o.fastq_split(data)
    w = [0] * nv.ST_WORDS
    w[nv.ST_N_LINES] = int((data == 10).sum())
    w[nv.ST_N_RECORDS] = r
    w[nv.ST_N_COMPLETE_BYTES], w[nv.ST_N_BASES], w[nv.ST_N_VALUES] = (int(x) for x in stats)
    w[nv.ST_BAD_HEADER_ENTRY] = w[nv.ST_BAD_PLUS_ENTRY] = nv.INT64_MAX
    w[nv.ST_BAD_BASE] = nv.INT64_MAX if bad is None else (bad[0] << 32) | bad[1]
    w[nv.ST_LAST_ROW_START] = int(starts[-1, 1]) + 1
    w[nv.ST_LAST_ROW_INDEX] = r
    return w


def count(data, enc_name):
    from bionumpy_b200 import ops
    mode, alphabet = ENCODINGS[enc_name]
    lut = torch.from_numpy(o.alphabet_lut(alphabet)).cuda() if mode == 3 else None
    hist, status = ops.chunk_kmer_count(torch.from_numpy(data).cuda(), K, BINS, enc_mode=mode, lut=lut)
    return hist.cpu().numpy(), status.cpu().tolist()


# ---- every row shape, all bytes valid ----------------------------------------------------------------------------------
def shapes_chunk():
    r = Records(31)
    rng = r.rng
    pairs = [(m, o16) for m in range(16) for o16 in range(16)]
    for _ in range(3):                    # 120 + m k-mers at every offset, shuffled: every chunk mixes them
        for i in rng.permutation(len(pairs)).tolist():
            m, o16 = pairs[i]
            r.add(READ + m, mod16=o16)
    for i in range(48):                   # bench-length rows (10 and 11 units) between rows with few or no k-mers
        r.add(READ, mod16=11 * i % 16)
        r.add(int(rng.integers(0, K)), mod16=int(rng.integers(16)))
        r.add(int(rng.integers(K, K + 48)), mod16=(7 * i + 3) % 16)
    for _ in range(3):                    # chunks in which no row has a k-mer: the walk has no block
        for _ in range(100):
            r.add(int(rng.integers(0, K)), mod16=int(rng.integers(16)))
        for L in (K - 1, K, K + 1, K + 15, K + 16, K + 17):
            r.add(L, mod16=int(rng.integers(16)))
    for g in range(3):                    # one long row among 31 short ones: a walk of 29 blocks
        for j in range(32):
            r.add(LONG if j == 7 + 9 * g else int(rng.integers(0, 60)), mod16=int(rng.integers(16)))
    r.filler(600, 400)
    return r.bytes()


def kernel_chunks(data):
    """Row indices of each 32-row chunk the kernel deals: rows 32c.. of the rows whose preceding newline is in a tile."""
    _, starts, _ = o.fastq_split(data)
    tile = (starts[:, 1] - 1) // TILE
    first = np.searchsorted(tile, tile)
    key = tile * 1024 + (np.arange(tile.size) - first) // 32
    return [np.flatnonzero(key == v) for v in np.unique(key)]


@gpu
@pytest.mark.parametrize("enc_name", list(ENCODINGS))
def test_every_row_shape_counts_like_the_oracle(enc_name):
    data = shapes_chunk()
    alphabet = ENCODINGS[enc_name][1]
    _, want, _ = c_oracle_hist(data, K, BINS, alphabet=alphabet.encode())
    hist, words = count(data, enc_name)
    assert np.array_equal(hist, want), (int(hist.sum()), int(want.sum()))
    assert words == expected_words(data, alphabet)


def test_shapes_chunk_covers_the_walk():
    """CPU check of the input: every (k-mer count mod 16, row end mod 16); kernel chunks that mix 10- and 11-unit rows
    with rows without a k-mer, chunks in which no row has a k-mer, and chunks with one long row."""
    data = shapes_chunk()
    _, starts, lens = o.fastq_split(data)
    s, L = starts[:, 1], lens[:, 1].astype(np.int64)
    npos = np.maximum(L - K + 1, 0)
    has = npos > 0
    ends = (s + L - 1) % 16
    assert {(int(a) % 16, int(b)) for a, b in zip(npos[has], ends[has])} == {(a, b) for a in range(16) for b in range(16)}
    units = (s + L - 1) // 16 - s // 16 + 1
    chunks = kernel_chunks(data)
    mixed = [c for c in chunks if {10, 11} <= set(units[c][L[c] == READ].tolist()) and not has[c].all()]
    assert len(mixed) >= 3
    assert sum(1 for c in chunks if c.size == 32 and not has[c].any()) >= 3
    assert sum(1 for c in chunks if L[c].max() == LONG and np.median(L[c]) < 60) >= 3
    assert L.max() < 512                           # every row ends inside the halo of the tile it starts in


# ---- bad bytes in the units the walk does not encode -------------------------------------------------------------------
TARGET = 5                                # the row with the bad byte: in the tile's first 32-row chunk


def bad_cases():
    """(label, target row length, its offset mod 16, length of the other rows, position of the bad byte)."""
    cases = []
    for o16 in range(16):
        last_unit = 16 * ((o16 + READ - 1) // 16) - o16      # first position of the row's last unit
        # 150-byte rows only: the walk has 8 blocks and encodes units 2..9; at offsets 11..15 the last unit (10) is past it
        cases.append(("last_byte", READ, o16, READ, READ - 1))
        cases.append(("last_unit", READ, o16, READ, last_unit))
    for L in (1, 17, K - 1):              # rows without a k-mer, among 150-byte rows and among rows without k-mers
        for o16 in (0, 9, 15):
            for others in (READ, 20):
                cases.append(("short_last_byte", L, o16, others, L - 1))
                if (o16 + L - 1) // 16 >= 2:
                    cases.append(("short_unit2", L, o16, others, 32 - o16))
    return cases


def bad_chunk(L, o16, others, pos, seed):
    r = Records(seed)
    for i in range(40):
        if i == TARGET:
            seq = bytearray(r.rng.choice(np.frombuffer(b"ACGT", dtype=np.uint8), size=L).tobytes())
            seq[pos] = ord("N")
            r.add(L, mod16=o16, seq=bytes(seq))
        else:
            r.add(others, mod16=int(r.rng.integers(16)))
    return r.bytes()


@gpu
@pytest.mark.parametrize("enc_name", list(ENCODINGS))
def test_bad_byte_past_the_walk(enc_name):
    alphabet = ENCODINGS[enc_name][1]
    for i, (label, L, o16, others, pos) in enumerate(bad_cases()):
        data = bad_chunk(L, o16, others, pos, seed=i)
        r, _, _ = c_oracle_hist(data, K, BINS, alphabet=alphabet.encode())
        _, starts, lens = o.fastq_split(data)
        flat = -1 - r
        row = int(np.searchsorted(np.cumsum(lens[:, 1]), flat, side="right"))
        bad = (row, flat - int(lens[:row, 1].sum()))
        assert bad == (TARGET, pos) and starts[TARGET, 1] % 16 == o16
        fixed = data.copy()
        fixed[starts[TARGET, 1] + pos] = ord("A")
        _, words = count(data, enc_name)
        assert words == expected_words(fixed, alphabet, bad), (label, L, o16, others, pos)
