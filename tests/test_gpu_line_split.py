"""bnpk_line_split (tile_kernel<0, ...>, cr_detect_kernel, finalize_status_kernel) against a plain NumPy split, at the
kernel's borders: 16384-byte tiles without halo, thread t owning bytes [64t, 64t + 64), 16-byte units, a three-ticket
prologue and newline windows of 1024 slots stepping by 1016.  Every starts / lens row below min(max_rows, n_records)
of every field line and the six status words are compared; for lines_per_entry 2 and 4 the expectation is also
checked against oracle.one_line_split."""
import numpy as np
import pytest
import torch

import reader_oracle as ro
from oracle import bnp_oracle as o

pytestmark = pytest.mark.gpu

TILE = 16384
NL, CR = 10, 13
SENT64, SENT32 = -0x5A5A5A5A5A5A5A5B, -0x2B2B2B2C
POISON = np.frombuffer(b"\n\r@+", dtype=np.uint8)


@pytest.fixture(scope="module")
def nv():
    from bionumpy_b200 import _native
    return _native


@pytest.fixture(scope="module")
def ops():
    from bionumpy_b200 import ops
    return ops


# ---- the expectation ---------------------------------------------------------------------------------------------
def expected(chunk, lpe, field_line, start_offset, header, check_plus, trim_cr):
    """(starts, lens, status dict) of a plain NumPy split; status as ops.ScanStatus interprets it."""
    nl = np.flatnonzero(chunk == NL)
    R = nl.size // lpe
    line_start = np.concatenate([[0], nl + 1]).astype(np.int64)   # start of line j = line_start[j]
    if trim_cr == 1:
        cr = chunk.size > 0
    elif trim_cr == 0 or R == 0:
        cr = False
    else:                                                         # the first lpe complete entries' header lines
        hdr_end = nl[0:min(lpe, R) * lpe:lpe]
        cr = bool(nl[0] >= 1 and np.any((hdr_end > line_start[0:min(lpe, R) * lpe:lpe]) & (chunk[hdr_end - 1] == CR)))
    idx = np.arange(R) * lpe + field_line
    starts = line_start[idx] + start_offset
    ends = nl[idx].astype(np.int64)
    if cr:
        ends = ends - ((ends > 0) & (chunk[np.maximum(ends - 1, 0)] == CR))
    lens = (ends - starts).astype(np.int32)
    bad_header = None
    if R == 0:
        bad_header = 0 if chunk.size and chunk[0] != header else None
    else:
        bad = np.flatnonzero(chunk[line_start[np.arange(R) * lpe]] != header)
        bad_header = int(bad[0]) if bad.size else None
    bad_plus = None
    if check_plus and lpe == 4 and R:
        bad = np.flatnonzero(chunk[line_start[np.arange(R) * lpe + 2]] != ord("+"))
        bad_plus = int(bad[0]) if bad.size else None
    st = dict(n_lines=int(nl.size), n_records=R, n_complete_bytes=int(nl[R * lpe - 1]) + 1 if R else 0,
              bad_header_entry=bad_header, bad_plus_entry=bad_plus, cr=bool(cr))
    return starts, lens, st


def cross_check_oracle(chunk, lpe, header, check_plus):
    """The plain split above is the reference's (one_line_split) for lines_per_entry 2 and 4 where that accepts, and
    a plain newline split for 1."""
    if lpe == 1:
        size, starts, lens = ro.plain_line_split(chunk)
        s, l, st = expected(chunk, 1, 0, 0, header, False, 0)
        assert st["n_complete_bytes"] == size and np.array_equal(s, starts) and np.array_equal(l, lens)
        return
    if np.count_nonzero(chunk == NL) < lpe:
        return
    try:
        size, starts, lens = o.one_line_split(chunk, lpe, header, (0,) * lpe, check_plus)
    except o.OracleFormatException:
        return
    for fl in range(lpe):
        s, l, st = expected(chunk, lpe, fl, 0, header, check_plus, -1)
        assert st["n_complete_bytes"] == size
        assert np.array_equal(s, starts[:, fl]) and np.array_equal(l, lens[:, fl])


# ---- the call ----------------------------------------------------------------------------------------------------
def view_of(chunk, offset=0):
    """chunk on the device at `offset` bytes past a 256-byte aligned allocation, poison behind it."""
    pad = 64
    buf = torch.empty(offset + chunk.size + pad, dtype=torch.uint8, device="cuda")
    assert buf.data_ptr() % 256 == 0
    host = np.empty(offset + chunk.size + pad, dtype=np.uint8)
    host[:] = POISON[np.arange(host.size) % 4]
    host[offset:offset + chunk.size] = chunk
    buf.copy_(torch.from_numpy(host))
    return buf[offset:offset + chunk.size]


def raw_split(nv, d, lpe, fl, so, header, check_plus, trim_cr, max_rows, extra=16):
    """bnpk_line_split through the C ABI with outputs `extra` rows longer than max_rows, pre-filled with a sentinel."""
    starts = torch.full((max_rows + extra,), SENT64, dtype=torch.int64, device="cuda")
    lens = torch.full((max_rows + extra,), SENT32, dtype=torch.int32, device="cuda")
    status = nv.new_status(d.device)
    ws = nv.workspace(max(d.numel(), 1), d.device)
    nv.check(nv.lib().bnpk_line_split(nv.ptr(d), d.numel(), lpe, fl, so, header, int(check_plus), trim_cr,
                                      nv.ptr(starts), nv.ptr(lens), max_rows, nv.ptr(status), nv.ptr(ws), ws.numel(),
                                      nv.stream_ptr()))
    return starts.cpu().numpy(), lens.cpu().numpy(), status


def check(ops, nv, chunk, lpe, header=ord("@"), check_plus=None, trim_crs=(-1,), offsets=(0,), fields=None,
          max_rows=None, start_offsets=None):
    chunk = np.asarray(chunk, dtype=np.uint8)
    if check_plus is None:
        check_plus = lpe == 4
    cross_check_oracle(chunk, lpe, header, check_plus)
    fields = range(lpe) if fields is None else fields
    for off in offsets:
        d = view_of(chunk, off)
        for trim_cr in trim_crs:
            for fl in fields:
                for so in (start_offsets or ((1,) if fl == 0 and lpe > 1 else (0,))):
                    s_want, l_want, st_want = expected(chunk, lpe, fl, so, header, check_plus, trim_cr)
                    R = st_want["n_records"]
                    for mr in ((R,) if max_rows is None else max_rows(R)):
                        s, l, status = raw_split(nv, d, lpe, fl, so, header, check_plus, trim_cr, mr)
                        st = ops.read_status(status)
                        got = {k: getattr(st, k) for k in st_want}
                        where = f"lpe={lpe} field={fl} so={so} trim_cr={trim_cr} off={off} max_rows={mr}"
                        assert got == st_want, where
                        k = min(mr, R)
                        assert np.array_equal(s[:k], s_want[:k]), where
                        assert np.array_equal(l[:k], l_want[:k]), where
                        assert np.all(s[mr:] == SENT64) and np.all(l[mr:] == SENT32), where


# ---- chunk builders ----------------------------------------------------------------------------------------------
def record_lines(rng, lpe, header, maxlen=60, eol=b""):
    L = int(rng.integers(0, maxlen + 1))
    seq = bytes(rng.choice(np.frombuffer(b"ACGT", dtype=np.uint8), size=L).tolist())
    h = bytes([header]) + b"r%d" % int(rng.integers(0, 1000))
    if lpe == 4:
        return [h + eol, seq + eol, b"+" + eol, b"I" * L + eol]
    if lpe == 2:
        return [h + eol, seq + eol]
    return [h + eol]


def join(lines):
    return np.frombuffer(b"".join(l + b"\n" for l in lines), dtype=np.uint8).copy()


def records_text(rng, n_bytes, lpe, header, maxlen=60, eol=b""):
    lines, size = [], 0
    while size < n_bytes:
        rec = record_lines(rng, lpe, header, maxlen, eol)
        lines += rec
        size += sum(len(x) + 1 for x in rec)
    return lines


def newline_at(rng, p, lpe, phase, header, after=3000, tail_lines=0):
    """Records with the newline of line `phase` of one entry at byte p, more records behind it, and `tail_lines` lines
    of an incomplete entry at the end."""
    lines, pos = [], 0
    while True:
        rec = record_lines(rng, lpe, header)
        n = sum(len(x) + 1 for x in rec)
        if pos + n > p - 80:
            break
        lines += rec
        pos += n
    rec = [bytes([header]), b"", b"+", b""][:lpe] if lpe > 1 else [bytes([header])]
    before = sum(len(x) + 1 for x in rec[:phase])
    need = p - pos - before
    first = rec[phase][:1]
    assert need >= len(first)
    rec[phase] = first + b"A" * (need - len(first))
    lines += rec
    lines += records_text(rng, after, lpe, header)
    lines += record_lines(rng, lpe, header)[:tail_lines]
    chunk = join(lines)
    assert chunk[p] == NL
    return chunk


# ---- cases -------------------------------------------------------------------------------------------------------
BORDERS = [63, 64, 127, 128, 1023, 1024, TILE - 1, TILE, TILE + 1, 2 * TILE - 1, 2 * TILE, 2 * TILE + 1, 3 * TILE - 1,
           3 * TILE, 3 * TILE + 1]


@pytest.mark.parametrize("lpe", [1, 2, 4])
@pytest.mark.parametrize("p", BORDERS)
def test_newline_on_thread_and_tile_borders(ops, nv, lpe, p):
    rng = np.random.default_rng(p * 7 + lpe)
    header = {1: ord("#"), 2: ord(">"), 4: ord("@")}[lpe]
    for phase in range(lpe):
        chunk = newline_at(rng, p, lpe, phase, header, tail_lines=phase % lpe)
        check(ops, nv, chunk, lpe, header, trim_crs=(-1, 0) if lpe > 1 else (0,))


@pytest.mark.parametrize("lpe", [2, 4])
def test_newline_at_every_offset_of_a_unit(ops, nv, lpe):
    rng = np.random.default_rng(lpe)
    for base in (TILE + 16 * 7, 2 * TILE - 16):
        for j in range(16):
            chunk = newline_at(rng, base + j, lpe, j % lpe, ord("@"), after=200)
            check(ops, nv, chunk, lpe, trim_crs=(-1,), fields=(1, lpe - 1))


@pytest.mark.parametrize("lpe", [2, 4])
def test_cr_before_a_tile_border(ops, nv, lpe):
    """'\\r' the last byte of a tile, its '\\n' the first byte of the next; CRLF everywhere."""
    rng = np.random.default_rng(11)
    for phase in range(lpe):
        lines = [l + b"\r" for l in records_text(rng, TILE - 2000, lpe, ord("@"))]
        pos = sum(len(x) + 1 for x in lines)
        rec = [b"@", b"", b"+", b""][:lpe]
        rec = [x + b"\r" for x in rec]
        before = sum(len(x) + 1 for x in rec[:phase])
        rec[phase] = rec[phase][:-1] + b"A" * (TILE - pos - before - len(rec[phase])) + b"\r"
        lines += rec + [l + b"\r" for l in records_text(rng, 2000, lpe, ord("@"))]
        chunk = join(lines)
        assert chunk[TILE - 1] == CR and chunk[TILE] == NL
        check(ops, nv, chunk, lpe, trim_crs=(-1, 0, 1))


@pytest.mark.parametrize("n_tiles", [1, 2, 3, 4])
@pytest.mark.parametrize("lpe", [1, 2, 4])
def test_tile_counts(ops, nv, n_tiles, lpe):
    rng = np.random.default_rng(n_tiles * 10 + lpe)
    for size in (n_tiles * TILE - 1, n_tiles * TILE, n_tiles * TILE - 300):
        if size <= 0:
            continue
        lines = records_text(rng, size, lpe, ord("@"))
        chunk = join(lines)[:size]
        check(ops, nv, chunk, lpe, trim_crs=(-1,) if lpe > 1 else (0,), offsets=(0, 5))


def test_more_tiles_than_the_resident_ctas_take_in_their_prologue(ops, nv):
    sm = int(nv.lib().bnpk_sm_count())
    n_rec = (3 * 4 * sm + 37) * TILE // 317 + 1
    chunk = np.concatenate([o.synthetic_fastq(0, n_rec), np.frombuffer(b"@tail\nACGT\n+\n", dtype=np.uint8)])
    assert chunk.size > 3 * 4 * sm * TILE
    check(ops, nv, chunk, 4, fields=(0, 1, 3))
    check(ops, nv, chunk, 2, header=ord("@"), check_plus=False, fields=(1,))


def dense_tile_chunk(k, unit, lead, tail=b"", tiles_before=1):
    """`tiles_before` tiles of `lead` records, then one tile holding exactly k newlines (repeats of `unit`, the
    rest a newline-free line), then `tail`."""
    per = unit.count(b"\n")
    body = unit * (k // per)
    if k % per:
        body += unit[: [i for i, c in enumerate(unit) if c == NL][k % per - 1] + 1]
    assert body.count(b"\n") == k and len(body) <= TILE
    pre = b"".join(l + b"\n" for l in lead)[: tiles_before * TILE]
    pre = pre + b"x" * (tiles_before * TILE - len(pre))
    filler = b"x" * (TILE - len(body))
    chunk = np.frombuffer(pre + filler + body + tail, dtype=np.uint8)
    assert np.count_nonzero(chunk[tiles_before * TILE:(tiles_before + 1) * TILE] == NL) == k
    return chunk


@pytest.mark.parametrize("k", [1023, 1024, 1025, 2040, 2041, 16384])
@pytest.mark.parametrize("kind", ["empty", "fastq", "fasta1"])
def test_newline_windows(ops, nv, k, kind):
    rng = np.random.default_rng(k)
    lpe, header, unit = {"empty": (4, ord("@"), b"\n"), "fastq": (4, ord("@"), b"@\n\n+\n\n"),
                         "fasta1": (1, ord(">"), b">\nA\nC\n")}[kind]
    lead = records_text(rng, 2 * TILE, lpe, header)
    if k == TILE and kind != "empty":
        pytest.skip("only empty lines fill a tile with newlines")
    for tail in (b"", b"@r\nACGT\n+\nII\n", b"@r\nACGT\n" * 40 + b"\n" * 1100):
        # the chunk's last complete entry ends in the dense tile's first, a middle or the last window, or later
        chunk = dense_tile_chunk(k, unit, lead, tail)
        check(ops, nv, chunk, lpe, header, check_plus=lpe == 4, trim_crs=(-1,) if lpe > 1 else (0,),
              fields=range(lpe) if lpe < 4 else (0, 1, 3))
    for cut in (3, 500, 1016 * 3 + 5):           # cut inside the dense tile: the last window is the one cut
        chunk = dense_tile_chunk(k, unit, lead)
        chunk = chunk[: chunk.size - cut]
        check(ops, nv, chunk, lpe, header, check_plus=lpe == 4, trim_crs=(-1,) if lpe > 1 else (0,),
              fields=(0, 1) if lpe > 1 else (0,))


@pytest.mark.parametrize("lpe", [2, 4])
def test_long_lines(ops, nv, lpe):
    rng = np.random.default_rng(3)
    for L in (TILE + 100, 3 * TILE + 5, 4 * TILE):
        head = records_text(rng, 500, lpe, ord("@"))
        rec = [b"@long", b"A" * L, b"+", b"I" * L][:lpe]
        check(ops, nv, join(head + rec + records_text(rng, 700, lpe, ord("@"))), lpe)
        # an incomplete tail that spans several tiles after the last complete entry
        check(ops, nv, join(head + rec[:lpe - 1]), lpe, max_rows=lambda R: (R, R + 1))
        check(ops, nv, np.concatenate([join(head), np.full(L, ord("A"), np.uint8)]), lpe)


@pytest.mark.parametrize("lpe", [1, 2, 4])
def test_views_at_every_offset(ops, nv, lpe):
    rng = np.random.default_rng(5)
    chunk = join(records_text(rng, 2 * TILE + 77, lpe, ord("@")))
    check(ops, nv, chunk, lpe, trim_crs=(-1,) if lpe > 1 else (0,), offsets=range(16), fields=(0, lpe - 1))
    check(ops, nv, chunk[:-1], lpe, trim_crs=(0,), offsets=range(16), fields=(lpe - 1,))   # poison right behind


@pytest.mark.parametrize("lpe", [1, 2, 4])
def test_max_rows(ops, nv, lpe):
    rng = np.random.default_rng(7)
    chunk = join(records_text(rng, 2 * TILE + 500, lpe, ord("@")) + [b"@x"])
    check(ops, nv, chunk, lpe, trim_crs=(-1,) if lpe > 1 else (0,),
          max_rows=lambda R: (0, 1, R // 2, R - 1, R, R + 1))


def test_start_offsets_and_header_chars(ops, nv):
    rng = np.random.default_rng(8)
    for header in (ord("@"), ord(">"), ord("#")):
        for lpe in (1, 2, 4):
            chunk = join(records_text(rng, TILE + 300, lpe, header))
            check(ops, nv, chunk, lpe, header, trim_crs=(0,), start_offsets=(0, 1))
    chunk = join(records_text(rng, TILE + 300, 4, ord("@")))
    chunk[np.flatnonzero(chunk == ord("+"))[3]] = ord("-")
    for cp in (True, False):
        check(ops, nv, chunk, 4, check_plus=cp, fields=(1,))


def entry_line_starts(chunk, lpe):
    nl = np.flatnonzero(chunk == NL)
    return np.concatenate([[0], nl + 1])[: (nl.size // lpe) * lpe: 1]


@pytest.mark.parametrize("lpe", [2, 4])
def test_validation(ops, nv, lpe):
    """A bad header or '+' on the first, an interior and the last complete entry, on tile borders, in a later window,
    two errors at once (the smaller entry wins) and an error in the incomplete tail (not reported)."""
    rng = np.random.default_rng(9)
    base = join(records_text(rng, 3 * TILE, lpe, ord("@"), maxlen=4) + record_lines(rng, lpe, ord("@"))[:lpe - 1])
    starts = entry_line_starts(base, lpe)
    R = starts.size // lpe
    tile1 = int(np.searchsorted(starts[::lpe], TILE))                # first entry starting at or after byte 16384
    later_window = int(np.searchsorted(np.flatnonzero(base == NL), TILE + 1500 * 4) // lpe)
    kinds = ["hdr"] + (["plus"] if lpe == 4 else [])
    for kind in kinds:
        line = 0 if kind == "hdr" else 2
        for entries in ([0], [R // 2], [R - 1], [tile1], [tile1 - 1], [later_window], [R // 2, 3], [R - 1, tile1],
                        [R]):
            chunk = base.copy()
            for e in entries:
                at = starts[e * lpe + line] if e < R else np.flatnonzero(base == NL)[R * lpe - 1] + 1
                chunk[at] = ord("-")
            check(ops, nv, chunk, lpe, fields=(1,))
    # a header char on a tile's first byte: an entry placed to start exactly there
    chunk = newline_at(rng, TILE - 1, lpe, lpe - 1, ord("@"))
    assert chunk[TILE] == ord("@")
    chunk[TILE] = ord("!")
    check(ops, nv, chunk, lpe, fields=(1,))


@pytest.mark.parametrize("lpe", [2, 4])
def test_carriage_returns(ops, nv, lpe):
    rng = np.random.default_rng(10)
    lines = records_text(rng, 2 * TILE, lpe, ord("@"))
    cases = {
        "headers_0_to_3": [i for i in range(0, 4 * lpe, lpe)],
        "line_16": [16],
        "every_line": list(range(len(lines))),
        "header_1_only": [lpe],
        "empty_after_trim": [1, lpe + 1],
    }
    for name, which in cases.items():
        ls = list(lines)
        for i in which:
            ls[i] = (b"" if name == "empty_after_trim" else ls[i]) + b"\r"
        check(ops, nv, join(ls), lpe, trim_crs=(-1, 0, 1), fields=range(lpe))


@pytest.mark.parametrize("lpe", [2, 4])
def test_carriage_return_only_in_the_incomplete_tail(ops, nv, lpe):
    """Fewer than lpe complete entries, and the first header ending in '\\r' belongs to the incomplete entry: the
    reference trims nothing (one_line_buffer.py:175-182 reads only the complete entries)."""
    rng = np.random.default_rng(12)
    for n_complete in range(0, lpe):
        for tail_lines in range(1, lpe):
            lines = []
            for _ in range(n_complete):
                lines += record_lines(rng, lpe, ord("@"))
            tail = record_lines(rng, lpe, ord("@"))[:tail_lines]
            tail[0] += b"\r"
            lines += tail
            for i in range(1, len(lines)):                   # every non-header line ends in '\r'
                if i % lpe:
                    lines[i] += b"\r"
            chunk = join(lines)
            check(ops, nv, chunk, lpe, trim_crs=(-1,))


def test_carriage_return_in_the_tail_of_the_fused_count(ops, nv):
    """The fused count decides '\\r' with the same kernel: the same chunk must count like the oracle."""
    text = b"@a\nACGTACGT\n+\nIIIIIIII\r\n@b\r\nACGTA"
    chunk = np.frombuffer(text, dtype=np.uint8)
    d = view_of(chunk)
    for k in (1, 3):
        hist, status = ops.chunk_kmer_count(d, k, 4 ** k)
        want, size, n_bases = o.fastq_chunk_kmer_counts(chunk, k, 4 ** k, False)
        st = ops.read_status(status)
        assert np.array_equal(hist.cpu().numpy(), want)
        assert st.n_complete_bytes == size and st.n_bases == n_bases and not st.cr


@pytest.mark.parametrize("lpe", [1, 2, 4])
def test_degenerate_chunks(ops, nv, lpe):
    for text in (b"", b"@", b"@abc", b"@" + b"A" * (TILE + 5), b"@a\n" * (lpe - 1), b"\n" * (lpe - 1)):
        chunk = np.frombuffer(text, dtype=np.uint8)
        if chunk.size == 0:
            d = torch.empty(0, dtype=torch.uint8, device="cuda")
            s, l, status = raw_split(nv, d, lpe, 0, 0, ord("@"), lpe == 4, -1, 0)
            st = ops.read_status(status)
            assert (st.n_lines, st.n_records, st.n_complete_bytes, st.bad_header_entry, st.bad_plus_entry, st.cr) == \
                (0, 0, 0, None, None, False)
            assert np.all(s == SENT64)
            continue
        check(ops, nv, chunk, lpe, trim_crs=(-1, 0, 1) if lpe > 1 else (0, 1), max_rows=lambda R: (0, 1))


def test_dispatcher_op_equals_ops(ops, nv):
    from bionumpy_b200 import torch_ops
    torch_ops.load()
    rng = np.random.default_rng(13)
    chunk = join(records_text(rng, 2 * TILE + 11, 4, ord("@")) + [b"@t\r", b"AC"])
    d = view_of(chunk, 3)
    R = np.count_nonzero(chunk == NL) // 4
    a = ops.line_split(d, 4, 3, 0, ord("@"), True, -1, max_rows=R)
    b = torch.ops.bnpk.line_split(d, 4, 3, 0, ord("@"), True, -1, R)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1]) and torch.equal(a[2], b[2])
