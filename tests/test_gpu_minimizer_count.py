"""The fused minimizer count (bnpk_chunk_kmer_count with window_size > 0) on every kernel route, against a plain window
minimum.

The expected values never come from the sliding-minimum scheme the kernels use (log-doubling shuffles, block minima):
every k-mer is hashed (sum_j code[i+j] * 4^j), every window takes the minimum of its window_size - k + 1 hashes with
`sliding_window_view(...).min(axis=-1)` (`oracle.get_minimizers`), or with the C oracle's ring minimum for the full-size
cases.  A CPU test pins that helper to the reference's literal formulation.

Inputs are built on purpose, not drawn at random: rows of the lengths where a window count changes (0, 1, k - 1, k,
window - 1, window, window + 1, k-mer counts at multiples of the window length +-1), rows at every byte offset mod 16,
rows at the staging and deferral thresholds of the kernels, rows that end at the last byte of a staged tile +-1, rows
longer than a tile, tiles with more newlines than the newline list holds, and 32-row chunks in which one long row
drives the warp-uniform decisions.  Every count goes into a histogram pre-filled with random values, and every status
word is checked."""
import numpy as np
import pytest
import torch

from oracle import bnp_oracle as o
from test_gpu_sliced_count import Input, PROFILE_ATTEMPTS, Route, _normalise, count_sliced, prefill, schedule
from test_oracle_goldens import c_oracle_hist

gpu = pytest.mark.gpu

TILE = 16384
WSM_SLOT = TILE + 512              # bytes a tile of the warp-specialised build stages (tile + halo)
TILE_STAGED = TILE + 2048          # bytes a tile of the register-staged tile kernel stages
ROW_MAX = 1024                     # longest row the warp-specialised row walk counts itself
MINZ_W = 12                        # longest window, in k-mers, of the warp-specialised minimizer build
HIST_AUTO, HIST_SMEM, HIST_GLOBAL = 0, 1, 2
ENC_ACGT, ENC_ACTG, ENC_LUT = 0, 1, 3
ALPHABET = {ENC_ACGT: "ACGT", ENC_ACTG: "ACTG", ENC_LUT: "ACTG"}

# The kernels a call must reach, as the profiler names them (template arguments normalised)
KERNELS = {
    "wsm": "bnpk::wsm::tile_ws_kernel<{enc}>",
    "tile_smem": "bnpk::tile_kernel<1, {enc}, true, true>",
    "tile_global": "bnpk::tile_kernel<1, {enc}, false, true>",
    "deferred": "bnpk::rows_kernel<4, {enc}, false, true>",        # RM_COUNT_MIN, global table, deferred rows
    "uncount": "bnpk::uncount_kernel<{enc}, true>",
}
COUNT_KERNELS = ("bnpk::ws::", "bnpk::wsm::", "bnpk::tma::", "bnpk::tile_kernel<", "bnpk::rows_kernel<",
                 "bnpk::uncount_kernel<")


def count_route(k, window, bins, hist_mode=HIST_AUTO, shift=0):
    """The kernel that counts the rows a tile holds (tile_ws_kernel.cu wsm_count_eligible, launch_count)."""
    smem = hist_mode != HIST_GLOBAL and bins <= 1 << 15
    if smem and bins <= 1 << 14 and window - k + 1 <= MINZ_W and shift == 0:
        return "wsm"
    return "tile_smem" if smem else "tile_global"


# ---- the oracle ---------------------------------------------------------------------------------------------------------
def window_minima(codes, lens, k, window):
    """Per row, the minimum of every window_size - k + 1 consecutive k-mer hashes (a plain window minimum)."""
    return o.get_minimizers(codes, lens, k, window)


def expect(data, lpe, k, window, bins, alphabet="ACGT"):
    """(hist, status words) of the reference path: split, sequence rows, encode, window minima, bincount(v % bins)."""
    size, starts, lens = (o.fastq_split if lpe == 4 else o.two_line_fasta_split)(data)
    L = lens[:, 1].astype(np.int64)
    codes = o.encode_flat(o.gather_rows(data, starts[:, 1], L), o.alphabet_lut(alphabet))
    vals, _ = window_minima(codes, L, k, window)
    n_values = int(np.maximum(L - window + 1, 0).sum())
    assert vals.size == n_values
    return np.bincount(vals % bins, minlength=bins), (starts.shape[0], size, int(L.sum()), n_values)


def bad_base_of(data, lpe, alphabet="ACGT"):
    """(row, position) of the first byte outside the alphabet, as the oracle raises it."""
    _, starts, lens = (o.fastq_split if lpe == 4 else o.two_line_fasta_split)(data)
    L = lens[:, 1].astype(np.int64)
    with pytest.raises(o.OracleEncodingError) as e:
        o.encode_flat(o.gather_rows(data, starts[:, 1], L), o.alphabet_lut(alphabet))
    ends = np.cumsum(L)
    row = int(np.searchsorted(ends, e.value.offset, side="right"))
    return row, int(e.value.offset - (ends[row] - L[row]))


# ---- inputs -------------------------------------------------------------------------------------------------------------
ACGT = np.frombuffer(b"ACGT", dtype=np.uint8)


class Records:
    """FASTQ (lpe 4) or two-line FASTA (lpe 2) text built record by record.  A record's sequence line can be put at a
    chosen byte (its header is padded to reach it) or at a chosen offset mod 16."""

    def __init__(self, seed, lpe=4, eol=b"\n", lower=0.3):
        self.rng, self.lpe, self.eol, self.lower = np.random.default_rng(seed), lpe, eol, lower
        self.parts, self.n, self.n_rec, self.rows = [], 0, 0, []

    def _seq(self, L):
        s = self.rng.choice(ACGT, size=L)
        return np.where(self.rng.random(L) < self.lower, s + 32, s).astype(np.uint8).tobytes()

    def _head_min(self):
        return 1 + len(b"r%d" % self.n_rec) + len(self.eol)

    def add(self, L, at=None, mod16=None, seq=None):
        """One record with L bases; returns (first byte of its sequence line, first byte of its quality line)."""
        name = (b"@" if self.lpe == 4 else b">") + b"r%d" % self.n_rec
        s0 = self.n + len(name) + len(self.eol)
        if mod16 is not None:
            at = s0 + (mod16 - s0) % 16
        if at is not None:
            assert at >= s0, (at, s0)
            name += b"x" * (at - s0)
            s0 = at
        seq = self._seq(L) if seq is None else seq
        rec = [name, self.eol, seq, self.eol]
        q0 = s0 + L + 2 * len(self.eol) + 1
        if self.lpe == 4:
            rec += [b"+", self.eol, self.rng.integers(33, 74, size=L, dtype=np.uint8).tobytes(), self.eol]
        self.parts += rec
        self.n += sum(len(p) for p in rec)
        self.n_rec += 1
        self.rows.append(seq)
        return s0, q0

    def filler(self, n, max_len):
        for L in self.rng.integers(0, max_len + 1, n).tolist():
            self.add(L)

    def place(self, at, L, max_len=120):
        """Short records up to byte `at`, then a record whose sequence line starts there."""
        rec_max = 16 + 2 * max_len + 4 * len(self.eol)
        while at - self.n > 2 * rec_max:
            self.add(int(self.rng.integers(0, max_len + 1)))
        return self.add(L, at=at)

    def end_line_at(self, tile, rel_newline):
        """A row that starts 40 bytes before the end of `tile` and whose '\\n' is byte `rel_newline` of the tile."""
        start = tile * TILE + TILE - 40
        return self.place(start, rel_newline - (TILE - 40) - len(self.eol) + 1)

    def bytes(self):
        return np.frombuffer(b"".join(self.parts), dtype=np.uint8).copy()


def edge_lengths(k, window):
    """Row lengths where a window count or a kernel decision changes."""
    W = window - k + 1
    lens = {0, 1, k - 1, k, window - 1, window, window + 1, ROW_MAX - 1, ROW_MAX, ROW_MAX + 1}
    for m in ((1, 2, 3, 5, 8) if W <= 100 else (1, 2, 3)):          # k-mer counts at multiples of W, +-1
        lens |= {m * W + d + k - 1 for d in (-1, 0, 1)}
    lens |= {160 + k - 1, 161 + k - 1, 176 + k - 1, 177 + k - 1}   # the longest row of a chunk: 10 / 11 blocks of 16
    return sorted(L for L in lens if L >= 0)


def edge_records(k, window, seed, lpe=4, eol=b"\n", dense=True):
    """The edge rows of (k, window), then rows at the staging / deferral thresholds and tile ends, long rows and a dense
    tile; returns the Records (more may be appended)."""
    r = Records(seed, lpe, eol)
    r.filler(40, 150)
    lens = edge_lengths(k, window)
    for i, L in enumerate(lens):                                    # each length at three offsets mod 16
        for o16 in (0, 7 + i % 8, 15):
            r.add(L, mod16=o16)
    for L in (192, 200, 208):                                       # rows touching 13 or 14 units: every offset
        for o16 in range(16):
            r.add(L, mod16=o16)
    short = min(window + 1, 60)
    for long_len in (160 + k - 1, 161 + k - 1, ROW_MAX, window + 1):   # 31 short rows and one long row, in every chunk
        for g in range(3):
            for j in range(32):
                r.add(long_len if j == (5 + 11 * g) % 32 else int(r.rng.integers(0, short + 1)))
    for L in (20000, 40000):                                        # longer than a tile
        r.add(L)
    tile = r.n // TILE + 2
    for rel in [WSM_SLOT - 2, WSM_SLOT - 1, WSM_SLOT, WSM_SLOT + 1,
                TILE_STAGED - 2, TILE_STAGED - 1, TILE_STAGED, TILE_STAGED + 1]:
        r.end_line_at(tile, rel)
        tile += 3
    if dense:                                                       # more than 1024 newlines in a tile
        r.filler(1000, min(window + 1, 24))
    r.filler(30, 400)
    return r


_inputs = {}


def edge_input(k, window, kind="lf"):
    """An edge chunk of (k, window) in one record style: "lf", "crlf", "fasta", or a last record truncated inside its
    sequence line ("trunc_seq") or its quality line ("trunc_qual", "trunc_qual_long": a row of 5000 bases, which the
    un-count walks in several segments)."""
    key = (k, window, kind)
    if key not in _inputs:
        seed = 1000 * k + window
        lpe, eol = (2, b"\n") if kind == "fasta" else (4, b"\r\n" if kind == "crlf" else b"\n")
        r = edge_records(k, window, seed, lpe, eol)
        if kind.startswith("trunc"):
            L = 5000 if kind == "trunc_qual_long" else window + 37
            s0, q0 = r.add(L)
            data = r.bytes()[: (s0 if kind == "trunc_seq" else q0) + L // 2].copy()
        else:
            data = r.bytes()
        _inputs[key] = (data, lpe)
    return _inputs[key]


# ---- one launch -------------------------------------------------------------------------------------------------------
def run(data, lpe, k, window, bins, hist_mode=HIST_AUTO, shift=0, enc=ENC_ACGT, seed=0):
    """One call of bnpk_chunk_kmer_count over the whole chunk, `shift` bytes into its buffer, into a pre-filled
    histogram.  Returns (counts added, ScanStatus)."""
    from bionumpy_b200 import ops
    src = torch.from_numpy(data).cuda()
    route = Route(k, bins, window, hist_mode, shift, ())
    inp = Input(data, lpe, "@" if lpe == 4 else ">", lpe == 4, None)
    lut = torch.from_numpy(o.alphabet_lut("ACTG")).cuda() if enc == ENC_LUT else None
    hist0 = prefill(bins, seed)
    hist, st = count_sliced(src, schedule("one_shot", src.numel()), route, inp, enc, lut, hist0=hist0)
    return (hist - hist0).cpu().numpy(), ops.ScanStatus(st)


def check(data, lpe, k, window, bins, hist_mode=HIST_AUTO, shift=0, enc=ENC_ACGT):
    want, words = expect(data, lpe, k, window, bins, ALPHABET[enc])
    got, st = run(data, lpe, k, window, bins, hist_mode, shift, enc, seed=window)
    if not np.array_equal(got, want):
        diff = np.flatnonzero(got != want)
        raise AssertionError(f"{diff.size} bins differ, first {diff[:5].tolist()}: got {got[diff[:5]].tolist()} "
                             f"want {want[diff[:5]].tolist()}; totals {int(got.sum())} / {int(want.sum())}")
    assert (st.n_records, st.n_complete_bytes, st.n_bases, st.n_values) == words
    assert not st.overflow and st.bad_base() is None
    assert st.bad_header_entry is None and st.bad_plus_entry is None


# ---- the oracle against the reference's formulation (CPU) -----------------------------------------------------------------
ORACLE_CASES = [(1, 1), (31, 31), (2, 3), (5, 7), (16, 27), (17, 29), (3, 33), (31, 62), (7, 39), (4, 67), (2, 101)]


@pytest.mark.parametrize("k,window", ORACLE_CASES)
def test_window_minimum_matches_the_reference_formulation(k, window):
    """W = window - k + 1 in {1, 1, 2, 3, 12, 13, 31, 32, 33, 64, 100} on small ragged rows around the window length."""
    rng = np.random.default_rng(window * 37 + k)
    lens = np.concatenate([[0, 1, k - 1, k, window - 1, window, window + 1], rng.integers(0, window + 40, 6)])
    lens = np.maximum(lens, 0)
    codes = rng.integers(0, 4, int(lens.sum())).astype(np.uint8)
    got, got_lens = window_minima(codes, lens, k, window)
    want, want_lens = o.get_minimizers_bruteforce(codes, lens, k, window)
    assert np.array_equal(got_lens, want_lens) and np.array_equal(got, want)


def test_edge_inputs_place_their_rows():
    """The builder puts rows where the cases need them: every offset mod 16, '\\n' at the chosen byte of a tile, and a
    tile with more than 1024 newlines."""
    r = Records(5)
    for o16 in range(16):
        s0, _ = r.add(200, mod16=o16)
        assert s0 % 16 == o16
    s0, _ = r.end_line_at(3, WSM_SLOT - 1)
    data = r.bytes()
    assert data[3 * TILE + WSM_SLOT - 1] == 10 and s0 == 3 * TILE + TILE - 40
    data, lpe = edge_input(31, 41)
    nl = np.flatnonzero(data == 10)
    assert np.bincount(nl // TILE).max() > 1024
    _, starts, lens = o.fastq_split(data)
    assert {0, 1, 30, 31, 40, 41, 42, 160 + 30, 161 + 30, 1023, 1024, 1025, 20000}.issubset(set(lens[:, 1].tolist()))
    nl_set = set(nl.tolist())
    for rel in (WSM_SLOT - 2, WSM_SLOT - 1, WSM_SLOT, WSM_SLOT + 1, TILE_STAGED - 2, TILE_STAGED + 1):
        # a row that starts in tile t (its '\n' before it in t) and ends at byte `rel` of t
        assert any(t * TILE + rel in nl_set and t * TILE + TILE - 41 in nl_set for t in range(data.size // TILE)), rel
    for kind, lines in (("trunc_seq", 1), ("trunc_qual", 3), ("trunc_qual_long", 3)):
        data, _ = edge_input(31, 41, kind)
        assert int((data == 10).sum()) % 4 == lines and data[-1] != 10


# ---- the cases, by the kernel they must reach ---------------------------------------------------------------------------
WSM_BINS = [64, 128, 256, 512, 1024, 2048, 4096, 8192, 1 << 14, 100, 12289]


def wsm_case(k, W):
    window = k + W - 1
    if k <= 2 and W % 2:
        bins = 4 ** k                                              # the exact table
    else:
        bins = WSM_BINS[(W + k) % len(WSM_BINS)]
    enc = ENC_ACTG if W == 7 else ENC_LUT if W == 10 else ENC_ACGT
    return window, bins, HIST_SMEM if W == 5 else HIST_AUTO, enc


WSM_CASES = [(k, W) for k in (1, 2, 15, 16, 17, 31) for W in range(1, MINZ_W + 1)]
TILE_WINDOWS = [13, 16, 31, 32, 33, 64, 100, "1024b"]              # k-mers per window; "1024b": window_size 1024
TILE_TABLES = {"smem": [(1 << 14, HIST_AUTO), ((1 << 14) + 1, HIST_AUTO), (30000, HIST_AUTO), (1 << 15, HIST_AUTO)],
               "global": [(1 << 20, HIST_AUTO), (1000003, HIST_AUTO), (1 << 14, HIST_GLOBAL), ((1 << 15) + 1, HIST_AUTO)]}
TILE_CASES = [(k, W, t) for k in (1, 16, 31) for W in TILE_WINDOWS for t in TILE_TABLES]


def tile_case(k, W, table):
    window = 1024 if W == "1024b" else k + W - 1
    i = TILE_WINDOWS.index(W)
    bins, mode = TILE_TABLES[table][(i + k) % 4]
    if k == 1 and W == 13 and table == "smem":
        bins = 4                                                    # the exact table
    enc = ENC_ACTG if W == 16 else ENC_LUT if W == 33 else ENC_ACGT
    return window, bins, mode, enc


@gpu
@pytest.mark.parametrize("k,W", WSM_CASES)
def test_wsm_window_sweep(k, W):
    """Every window of the warp-specialised build (1..12 k-mers) at k = 1, 2, 15, 16, 17 (where the hash's high word
    starts) and 31, on the edge rows, the deferred rows and the dense tile."""
    window, bins, mode, enc = wsm_case(k, W)
    assert count_route(k, window, bins, mode) == "wsm"
    data, lpe = edge_input(k, window)
    check(data, lpe, k, window, bins, mode, enc=enc)


@gpu
@pytest.mark.parametrize("k,W,table", TILE_CASES)
def test_tile_window_sweep(k, W, table):
    """Windows of 13 k-mers and more: the warp-shuffle branch of row_count (<= 32) and its per-lane branch (> 32, up
    to window_size 1024), on the shared-memory table and on the global one; long rows go to the deferred pass."""
    window, bins, mode, enc = tile_case(k, W, table)
    assert count_route(k, window, bins, mode) == "tile_" + table
    data, lpe = edge_input(k, window)
    check(data, lpe, k, window, bins, mode, enc=enc)


UNALIGNED_CASES = [(15, 20, 1), (15, 20, 8), (31, 42, 15), (16, 27, 3), (5, 60, 9)]


@gpu
@pytest.mark.parametrize("k,window,shift", UNALIGNED_CASES)
def test_unaligned_chunk(k, window, shift):
    """A chunk 1..15 bytes off 16-byte alignment goes to the tile kernel, whatever its window."""
    assert count_route(k, window, 1 << 14, HIST_AUTO, shift) == "tile_smem"
    data, lpe = edge_input(k, window)
    check(data, lpe, k, window, 1 << 14, shift=shift)


RECORD_ROUTES = {"wsm_w11": (31, 41, 1 << 14, HIST_AUTO), "wsm_w12": (16, 27, 4096, HIST_AUTO),
                 "tile_w13": (21, 33, 1 << 14, HIST_AUTO), "tile_w64": (16, 79, 1 << 20, HIST_AUTO),
                 "tile_1024b": (31, 1024, 30000, HIST_AUTO)}
RECORD_KINDS = ["crlf", "fasta", "trunc_seq", "trunc_qual", "trunc_qual_long"]


@gpu
@pytest.mark.parametrize("route", list(RECORD_ROUTES))
@pytest.mark.parametrize("kind", RECORD_KINDS)
def test_records(kind, route):
    """CRLF, two-line FASTA, and a last record cut inside its sequence line or inside its quality line (the row was
    counted; the un-count takes its windows back)."""
    k, window, bins, mode = RECORD_ROUTES[route]
    data, lpe = edge_input(k, window, kind)
    check(data, lpe, k, window, bins, mode)


BAD_ROUTES = {"wsm": (31, 41, 1 << 14), "wsm_w12": (31, 42, 1 << 14), "tile": (31, 43, 1 << 14),
              "tile_global": (31, 70, 1 << 20)}


@gpu
@pytest.mark.parametrize("route", list(BAD_ROUTES))
@pytest.mark.parametrize("where", ["short_row", "tail0", "tail15", "tail29", "staged_tail"])
def test_bad_base(route, where):
    """A bad base in a row shorter than the window (no window counted, still reported), and in the last k - 1 bytes of
    a long row (past the last window; unstaged in the warp-specialised build) or of a staged one.  The status must
    name the oracle's (row, position)."""
    k, window, bins = BAD_ROUTES[route]
    short = where in ("short_row", "staged_tail")                   # every row of the chunk is staged
    r = Records(7)
    r.filler(200, 150 if short else 300)
    if where == "short_row":
        L, pos = window - 2, window // 2
    elif where == "staged_tail":
        L, pos = 150, 150 - 5
    else:
        L, pos = 600, 600 - 1 - int(where[4:])
    s0, _ = r.add(L, mod16=11)
    r.filler(200, 150 if short else 300)
    data = r.bytes()
    data[s0 + pos] = ord("N")
    want = bad_base_of(data, 4)
    assert want[1] == pos
    got, st = run(data, 4, k, window, bins)
    assert st.bad_base() == want
    assert not st.overflow


# ---- every route, once, through the profiler ---------------------------------------------------------------------------
PROFILED = [  # (case, k, window, bins, hist_mode, shift, enc)
    ("wsm", 15, 20, 1 << 14, HIST_AUTO, 0, ENC_ACGT),
    ("wsm_lut", 7, 18, 100, HIST_SMEM, 0, ENC_LUT),
    ("tile_w13", 16, 28, 1 << 14, HIST_AUTO, 0, ENC_ACGT),
    ("tile_bins_2^15", 15, 20, 30000, HIST_AUTO, 0, ENC_ACGT),
    ("tile_unaligned", 15, 20, 1 << 14, HIST_AUTO, 5, ENC_ACGT),
    ("tile_global", 15, 20, 1 << 20, HIST_AUTO, 0, ENC_ACGT),
    ("tile_hist_global", 15, 20, 1 << 14, HIST_GLOBAL, 0, ENC_ACTG),
    ("tile_w1024b", 31, 1024, 1 << 14, HIST_AUTO, 0, ENC_ACGT),
]


def test_cases_cover_every_route():
    """The parametrised cases reach every count route; long rows and truncated records (deferred pass, un-count) are
    exercised on each."""
    seen = {count_route(k, *wsm_case(k, W)[:3]) for k, W in WSM_CASES}
    seen |= {count_route(k, *tile_case(k, W, t)[:3]) for k, W, t in TILE_CASES}
    seen |= {count_route(k, w, 1 << 14, HIST_AUTO, s) for k, w, s in UNALIGNED_CASES}
    assert seen == {"wsm", "tile_smem", "tile_global"}
    assert {count_route(*r) for r in RECORD_ROUTES.values()} == {"wsm", "tile_smem", "tile_global"}
    assert {count_route(*c[1:6]) for c in PROFILED} == {"wsm", "tile_smem", "tile_global"}
    assert max(edge_lengths(31, 41)) > ROW_MAX and max(edge_lengths(1, 1024)) > ROW_MAX


@gpu
def test_each_case_reaches_its_kernel():
    """Each profiled case launches its count kernel, the minimizer build of the deferred pass and of the un-count,
    and no other count kernel.  The profiler can drop records late in a long process, so a session that lacks a kernel
    is repeated, up to PROFILE_ATTEMPTS sessions per case."""
    from torch.profiler import profile, ProfilerActivity
    any_kernel = False
    for name, k, window, bins, mode, shift, enc in PROFILED:
        data, lpe = edge_input(k, window)
        want = {KERNELS[r].format(enc=enc) for r in (count_route(k, window, bins, mode, shift), "deferred", "uncount")}
        sessions = []
        for _ in range(PROFILE_ATTEMPTS):
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                run(data, lpe, k, window, bins, mode, shift, enc)
                torch.cuda.synchronize()
            names = {_normalise(e.key) for e in prof.key_averages()}
            any_kernel |= any("bnpk::" in n for n in names)
            launched = {n for n in names if any(c in n for c in COUNT_KERNELS)}
            assert all(any(w in n for w in want) for n in launched), (name, sorted(launched), sorted(want))
            sessions.append(sorted(launched))
            if all(any(w in n for n in names) for w in want):
                break
        else:
            if not any_kernel:
                pytest.skip("the profiler recorded no CUDA kernels")
            raise AssertionError((name, sorted(want), sessions))


# ---- full size: the bench's record shape --------------------------------------------------------------------------------
FULL_CASES = [(1_000_000, 31, 41, 1 << 14), (1_000_000, 31, 41, 1 << 20), (200_000, 21, 33, 1 << 14)]


@gpu
@pytest.mark.parametrize("n_reads,k,window,bins", FULL_CASES)
def test_full_size_synthetic_reads(n_reads, k, window, bins):
    """Synthetic 150 bp reads (the benchmark's records) against the C oracle, bit for bit: k = 31, window 41 into 2^14
    bins (warp-specialised) and into 2^20 bins (tile kernel, global table); k = 21, window 33 (13 k-mers, tile kernel)."""
    from bionumpy_b200 import ops
    host = o.synthetic_fastq(0, n_reads)
    n_rec, want, stats = c_oracle_hist(host, k, bins, window)
    assert n_rec == n_reads
    chunk = ops.synth_fastq(n_reads)
    hist0 = prefill(bins, 3)
    hist, status = ops.chunk_kmer_count(chunk, k, bins, hist0.clone(), window)
    st = ops.read_status(status)
    assert np.array_equal((hist - hist0).cpu().numpy(), want)
    assert (st.n_records, st.n_complete_bytes, st.n_bases, st.n_values) == (n_reads, stats[0], stats[1], stats[2])
    assert st.n_values == n_reads * (150 - window + 1)
    assert not st.overflow and st.bad_base() is None


# ---- the public API ------------------------------------------------------------------------------------------------------
API_CASES = [(15, 26), (15, 27), (11, 60)]                         # 12, 13 and 50 k-mers per window


def _api_file(tmp_path, k, window):
    r = Records(k + window)
    lens = r.rng.integers(1, 401, 400)
    lens[300] = 40000                                               # cut into pieces on the row route
    for L in lens.tolist():
        r.add(L)
    path = tmp_path / "reads.fq"
    path.write_bytes(r.bytes().tobytes())
    return path, [s.decode() for s in r.rows]


@gpu
@pytest.mark.parametrize("k,window", API_CASES)
def test_public_count_kmers_hashed(tmp_path, k, window):
    """count_kmers_hashed on a chunk read with bnp.open (the fused count) equals the same call on a detached copy of
    the rows (the row kernels, with the 40000-base row cut into pieces) and the oracle."""
    import bionumpy_b200 as bnp
    from bionumpy_b200.rows import LONG_ROW, RowView
    path, strings = _api_file(tmp_path, k, window)
    B = 1 << 14
    seq = bnp.open(str(path)).read().sequence
    assert RowView(seq).chunk_buffer is not None
    detached = bnp.as_encoded_array(strings)
    assert RowView(detached).chunk_buffer is None and max(map(len, strings)) > LONG_ROW + window
    fused = bnp.count_kmers_hashed(seq, k, B, window_size=window).cpu().numpy()
    rows = bnp.count_kmers_hashed(detached, k, B, window_size=window).cpu().numpy()
    want, _ = expect(np.fromfile(path, dtype=np.uint8), 4, k, window, B)
    assert np.array_equal(fused, want) and np.array_equal(rows, want)


@gpu
@pytest.mark.parametrize("window", [1025, 10])
def test_public_bad_window_raises_before_launch(tmp_path, window):
    """window_size 1025, or smaller than k, raises AssertionError on both routes before any count kernel (at most the
    status block's initialisation runs) and leaves the rows as they were."""
    import bionumpy_b200 as bnp
    from bionumpy_b200 import _native as nv
    from bionumpy_b200.rows import RowView
    path, strings = _api_file(tmp_path, 15, 40)
    seq = bnp.open(str(path)).read().sequence
    detached = bnp.as_encoded_array(strings)
    for rows in (seq, detached):
        before = RowView(rows).base.clone()
        torch.cuda.synchronize()
        launches = nv.lib().bnpk_launch_count()
        with pytest.raises(AssertionError):
            bnp.count_kmers_hashed(rows, 15, 1 << 14, window_size=window)
        torch.cuda.synchronize()
        assert nv.lib().bnpk_launch_count() - launches <= 1
        assert torch.equal(RowView(rows).base, before)
