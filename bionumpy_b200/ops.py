"""Tensor-level wrappers over the C-ABI (include/bnpk.h).  Everything here runs on the current CUDA stream of the device
of the op's tensors; every tensor the library gets is checked by ``_pointer`` before anything is allocated or launched.
These are the operator-level mirror of the reference functions named in include/bnpk.h."""
import ctypes
import functools

import torch

from . import _native as nv
from ._native import check, lib, ptr, stream_ptr


class ArgumentError(TypeError, ValueError):
    """A tensor argument of the wrong dtype or element count: a TypeError and a ValueError, so either catches it."""


def _pointer(t, name="tensor", dtype=None, n=None, at_least=0, optional=False, host=False):
    """The pointer the library gets for the tensor argument ``name``: a contiguous tensor on a CUDA device (on the host
    with ``host``) of ``dtype``, with exactly ``n`` or at least ``at_least`` elements; None is a null pointer when
    ``optional``.  Reads tensor metadata only: no device work, no allocation, no synchronisation."""
    if t is None and optional:
        return ptr(None)
    if not isinstance(t, torch.Tensor) or t.is_cuda == host:
        if host:
            raise TypeError(f"{name} must be a host tensor")
        raise nv.NativeLibraryError(f"{name} must be a CUDA tensor: bionumpy_b200 has no CPU fallback")
    if not t.is_contiguous():
        raise ValueError(f"{name} must be contiguous")
    if dtype is not None and t.dtype != dtype:
        raise ArgumentError(f"{name} must be {dtype}, not {t.dtype}")
    if t.numel() != (t.numel() if n is None else n) or t.numel() < at_least:
        raise ArgumentError(f"{name} must have {f'at least {at_least}' if n is None else n} elements, not {t.numel()}")
    return ptr(t)


def _lut(t):
    """An optional table of 256 uint8: the kernels read all of it."""
    return _pointer(t, "lut", torch.uint8, n=256, optional=True)


def _status(t, optional=True):
    """A status block: int64, at least ST_WORDS words."""
    return _pointer(t, "status", torch.int64, at_least=nv.ST_WORDS, optional=optional)


def _tensors(x):
    """The tensors of an argument, inside lists and tuples too (writer fields, columns, contigs)."""
    if isinstance(x, torch.Tensor):
        return [x]
    return [t for y in x for t in _tensors(y)] if isinstance(x, (list, tuple)) else []


def _on_device(fn):
    """Run an op with the device of its first CUDA tensor argument current (kernels launch on the current device's
    current stream) and check that every CUDA tensor argument, inside lists and tuples too, lives there."""
    @functools.wraps(fn)
    def wrapper(*args, **kwargs):
        tensors = [t for t in _tensors(list(args) + list(kwargs.values())) if t.is_cuda]
        if not tensors:
            return fn(*args, **kwargs)
        dev = tensors[0].device
        for t in tensors:
            if t.device != dev:
                raise ValueError(f"{fn.__name__}: tensors on different devices ({t.device} and {dev})")
        with torch.cuda.device(dev):
            return fn(*args, **kwargs)
    return wrapper


class ScanStatus:
    """Host copy of the device status block (bnpk.h BNPK_ST_*)."""

    def __init__(self, words):
        self.words = [int(w) for w in words]

    n_lines = property(lambda s: s.words[nv.ST_N_LINES])
    n_records = property(lambda s: s.words[nv.ST_N_RECORDS])
    n_complete_bytes = property(lambda s: s.words[nv.ST_N_COMPLETE_BYTES])
    n_bases = property(lambda s: s.words[nv.ST_N_BASES])
    n_values = property(lambda s: s.words[nv.ST_N_VALUES])
    n_long_rows = property(lambda s: s.words[nv.ST_N_LONG_ROWS])
    cr = property(lambda s: bool(s.words[nv.ST_CR]))
    overflow = property(lambda s: bool(s.words[nv.ST_OVERFLOW]))

    @property
    def bad_header_entry(self):
        v = self.words[nv.ST_BAD_HEADER_ENTRY]
        return None if v == nv.INT64_MAX or v >= max(self.n_records, 1) and v != 0 else v

    @property
    def bad_plus_entry(self):
        v = self.words[nv.ST_BAD_PLUS_ENTRY]
        return None if v == nv.INT64_MAX or v >= self.n_records else v

    def bad_base(self, n_rows=None):
        """(row, position) of the first byte outside the alphabet, or None."""
        v = self.words[nv.ST_BAD_BASE]
        if v == nv.INT64_MAX:
            return None
        row, pos = v >> 32, v & 0xFFFFFFFF
        if n_rows is not None and row >= n_rows:
            return None
        return row, pos


def read_status(status_t) -> ScanStatus:
    return ScanStatus(status_t.cpu().tolist())   # synchronises the stream


@_on_device
def reset_status(status):
    """Initialise a status block (int64, at least ST_WORDS words) again in place.  Returns it."""
    check(lib().bnpk_status_init(_status(status, optional=False), stream_ptr()))
    return status


@_on_device
def count_byte(chunk, value: int) -> int:
    chunk_p = _pointer(chunk, "chunk", torch.uint8)
    out = torch.empty(1, dtype=torch.int64, device=chunk.device)
    check(lib().bnpk_count_byte(chunk_p, chunk.numel(), value, _pointer(out), stream_ptr()))
    return int(out.item())


@_on_device
def line_split(chunk, lines_per_entry=4, field_line=1, start_offset=0, header_char=ord("@"), check_plus=True,
               trim_cr=-1, max_rows=None):
    """K1.  Returns (starts int64[R'], lens int32[R'], status tensor).  R' = max_rows (default: the
    exact number of lines / lines_per_entry, obtained with one census pass)."""
    chunk_p = _pointer(chunk, "chunk", torch.uint8)
    n, dev = chunk.numel(), chunk.device
    if max_rows is None:
        max_rows = count_byte(chunk, 10) // lines_per_entry
    starts = torch.empty(max_rows, dtype=torch.int64, device=dev)
    lens = torch.empty(max_rows, dtype=torch.int32, device=dev)
    status = nv.new_status(dev)
    ws = nv.workspace(n, dev)
    check(lib().bnpk_line_split(chunk_p, n, lines_per_entry, field_line, start_offset, header_char, int(check_plus),
                                trim_cr, _pointer(starts), _pointer(lens), max_rows, _pointer(status), _pointer(ws),
                                ws.numel(), stream_ptr()))
    return starts, lens, status


def _hist(hist, n_bins, device):
    """The caller's histogram (int64, a bin for every bin below n_bins the kernels add to) or a zeroed one."""
    if hist is None:
        return torch.zeros(n_bins, dtype=torch.int64, device=device)
    _pointer(hist, "hist", torch.int64, at_least=n_bins)
    return hist


@_on_device
def chunk_kmer_count(chunk, k, n_bins, hist=None, window_size=0, lines_per_entry=4, header_char=ord("@"),
                     check_plus=True, trim_cr=-1, enc_mode=nv.ENC_ASCII_ACGT, lut=None, hist_mode=nv.HIST_AUTO,
                     status=None):
    """K6 on a device-resident chunk.  Accumulates into ``hist`` (int64[n_bins]); returns
    (hist, status tensor)."""
    chunk_p, lut_p, _ = _pointer(chunk, "chunk", torch.uint8), _lut(lut), _status(status)
    n, dev = chunk.numel(), chunk.device
    hist = _hist(hist, n_bins, dev)
    status = nv.new_status(dev) if status is None else status
    ws = nv.workspace(n, dev)
    check(lib().bnpk_chunk_kmer_count(chunk_p, n, 0, n, 1, lines_per_entry, header_char, int(check_plus), trim_cr,
                                      enc_mode, lut_p, k, window_size, n_bins, hist_mode, _pointer(hist),
                                      _pointer(status), _pointer(ws), ws.numel(), stream_ptr()))
    return hist, status


@_on_device
def row_offsets(lens, shrink=0):
    """int64[R+1] exclusive prefix sums of max(lens - shrink, 0)."""
    lens_p, n = _pointer(lens, "lens", torch.int32), lens.numel()
    out = torch.empty(n + 1, dtype=torch.int64, device=lens.device)
    ws = nv.workspace(max(n, 1), lens.device)
    check(lib().bnpk_row_offsets(lens_p, n, shrink, _pointer(out), _pointer(ws), ws.numel(), stream_ptr()))
    return out


def _ragged_out(lens, shrink, offsets, total, dtype):
    """The flat output of a row op and its row offsets: max(lens - shrink, 0) values per row unless ``offsets``
    (int64[R+1]) are given, ``total`` values (default offsets[-1])."""
    if offsets is None:
        offsets = row_offsets(lens, shrink)
    if total is None:
        total = int(offsets[-1].item())
    return torch.empty(total, dtype=dtype, device=lens.device), offsets


def _rows_args(base, starts, lens, lut=None, offsets=None, status=None):
    """Check the rows of a row op (base uint8, starts int64 and lens int32, one length per start), its optional lut,
    output offsets (int64, one per row and the total) and status block.  Returns the head of every bnpk_rows_* call,
    (base, base bytes, starts, lens, rows), and the lut's pointer."""
    head = (_pointer(base, "base", torch.uint8), base.numel(), _pointer(starts, "starts", torch.int64),
            _pointer(lens, "lens", torch.int32, n=starts.numel()), starts.numel())
    _pointer(offsets, "offsets", torch.int64, at_least=starts.numel() + 1, optional=True)
    _status(status)
    return head, _lut(lut)


@_on_device
def rows_encode(base, starts, lens, enc_mode, lut=None, offsets=None, status=None, total=None):
    head, lut_p = _rows_args(base, starts, lens, lut, offsets, status)
    out, offsets = _ragged_out(lens, 0, offsets, total, torch.uint8)
    status = nv.new_status(base.device) if status is None else status
    check(lib().bnpk_rows_encode(*head, enc_mode, lut_p, _pointer(offsets), _pointer(out), _pointer(status),
                                 stream_ptr()))
    return out, offsets, status


@_on_device
def rows_kmer_hash(base, starts, lens, enc_mode, k, lut=None, offsets=None, status=None, total=None):
    head, lut_p = _rows_args(base, starts, lens, lut, offsets, status)
    out, offsets = _ragged_out(lens, k - 1, offsets, total, torch.int64)
    status = nv.new_status(base.device) if status is None else status
    check(lib().bnpk_rows_kmer_hash(*head, enc_mode, lut_p, k, _pointer(offsets), _pointer(out), _pointer(status),
                                    stream_ptr()))
    return out, offsets, status


@_on_device
def rows_generic_hash(base, starts, lens, alphabet_size, k, lut=None, offsets=None, status=None, total=None):
    """sum_j code[i+j] * alphabet_size^j for alphabets that are not four letters (K3')."""
    head, lut_p = _rows_args(base, starts, lens, lut, offsets, status)
    out, offsets = _ragged_out(lens, k - 1, offsets, total, torch.int64)
    status = nv.new_status(base.device) if status is None else status
    check(lib().bnpk_rows_generic_hash(*head, lut_p, alphabet_size, k, _pointer(offsets), _pointer(out),
                                       _pointer(status), stream_ptr()))
    return out, offsets, status


@_on_device
def rows_minimizers(base, starts, lens, enc_mode, k, window_size, lut=None, offsets=None, status=None, total=None):
    head, lut_p = _rows_args(base, starts, lens, lut, offsets, status)
    out, offsets = _ragged_out(lens, window_size - 1, offsets, total, torch.int64)
    status = nv.new_status(base.device) if status is None else status
    check(lib().bnpk_rows_minimizers(*head, enc_mode, lut_p, k, window_size, _pointer(offsets), _pointer(out),
                                     _pointer(status), stream_ptr()))
    return out, offsets, status


@_on_device
def rows_kmer_count(base, starts, lens, enc_mode, k, n_bins, window_size=0, lut=None, hist=None,
                    hist_mode=nv.HIST_AUTO, status=None):
    head, lut_p = _rows_args(base, starts, lens, lut, status=status)
    hist = _hist(hist, n_bins, base.device)
    status = nv.new_status(base.device) if status is None else status
    check(lib().bnpk_rows_kmer_count(*head, enc_mode, lut_p, k, window_size, n_bins, hist_mode, _pointer(hist),
                                     _pointer(status), stream_ptr()))
    return hist, status


@_on_device
def rows_reverse_complement(base, starts, lens, lut, offsets=None, total=None):
    """get_reverse_complement on a ragged view: out row r = lut[row r backwards] (uint8, contiguous rows)."""
    head, lut_p = _rows_args(base, starts, lens, lut, offsets)
    out, offsets = _ragged_out(lens, 0, offsets, total, torch.uint8)
    check(lib().bnpk_rows_reverse_complement(*head, lut_p, _pointer(offsets), _pointer(out), stream_ptr()))
    return out, offsets


@_on_device
def rows_kmer_hash_canonical(base, starts, lens, enc_mode, k, complement_xor, lut=None, offsets=None, status=None,
                             total=None):
    """EXTENSION: min(h, hash of the reverse complement) for every k-mer (K3 with a second strand)."""
    head, lut_p = _rows_args(base, starts, lens, lut, offsets, status)
    out, offsets = _ragged_out(lens, k - 1, offsets, total, torch.int64)
    status = nv.new_status(base.device) if status is None else status
    check(lib().bnpk_rows_kmer_hash_canonical(*head, enc_mode, lut_p, k, complement_xor, _pointer(offsets),
                                              _pointer(out), _pointer(status), stream_ptr()))
    return out, offsets, status


@_on_device
def rows_kmer_count_canonical(base, starts, lens, enc_mode, k, complement_xor, n_bins, lut=None, hist=None,
                              hist_mode=nv.HIST_AUTO, status=None):
    head, lut_p = _rows_args(base, starts, lens, lut, status=status)
    hist = _hist(hist, n_bins, base.device)
    status = nv.new_status(base.device) if status is None else status
    check(lib().bnpk_rows_kmer_count_canonical(*head, enc_mode, lut_p, k, complement_xor, n_bins, hist_mode,
                                               _pointer(hist), _pointer(status), stream_ptr()))
    return hist, status


def _table_args(keys, counts, n_used):
    """(keys, counts, slots, n_used) of an exact k-mer table: int64 keys and counts of one length, an int64[1] count."""
    keys_p = _pointer(keys, "keys", torch.int64)
    return (keys_p, _pointer(counts, "counts", torch.int64, n=keys.numel()), keys.numel(),
            _pointer(n_used, "n_used", torch.int64, n=1))


@_on_device
def rows_kmer_table_insert(base, starts, lens, enc_mode, k, keys, counts, n_used, complement_xor=0, lut=None,
                           status=None):
    """EXTENSION: insert every k-mer of the rows (canonical ones when complement_xor != 0) into the exact table
    (keys, counts: int64[C], C a power of two, free slot = key -1); n_used (int64[1]) grows by the slots claimed.
    Returns the status tensor."""
    head, lut_p = _rows_args(base, starts, lens, lut, status=status)
    table = _table_args(keys, counts, n_used)
    status = nv.new_status(base.device) if status is None else status
    check(lib().bnpk_rows_kmer_table_insert(*head, enc_mode, lut_p, k, complement_xor, *table, _pointer(status),
                                            stream_ptr()))
    return status


@_on_device
def kmer_table_rehash(keys, counts, new_keys, new_counts, n_used, status=None):
    """Re-insert every (key, count) of a table into a cleared one (growth); n_used grows by the slots claimed there."""
    old, new, _ = _table_args(keys, counts, n_used), _table_args(new_keys, new_counts, n_used), _status(status)
    status = nv.new_status(keys.device) if status is None else status
    check(lib().bnpk_kmer_table_rehash(*old[:3], *new, _pointer(status), stream_ptr()))
    return status


def _pwm_args(matrix):
    """(alphabet size, matrix, motif length) of a float64 [motif_len, alphabet_size] matrix."""
    matrix_p = _pointer(matrix, "matrix", torch.float64)
    if matrix.dim() != 2:
        raise TypeError("matrix must be float64 of shape [motif_len, alphabet_size]")
    return matrix.shape[1], matrix_p, matrix.shape[0]


@_on_device
def rows_pwm_scores(base, starts, lens, enc_mode, matrix, lut=None, tail=False, offsets=None, status=None, total=None):
    """K7: motif scores of every window of the rows (every position with ``tail``), float64, in column order.
    ``matrix`` is [motif_len, alphabet_size] on the device.  Returns (scores, offsets, status)."""
    (head, lut_p), pwm = _rows_args(base, starts, lens, lut, offsets, status), _pwm_args(matrix)
    out, offsets = _ragged_out(lens, 0 if tail else max(matrix.shape[0] - 1, 0), offsets, total, torch.float64)
    status = nv.new_status(base.device) if status is None else status
    check(lib().bnpk_rows_pwm_scores(*head, enc_mode, lut_p, *pwm, int(tail), _pointer(offsets), _pointer(out),
                                     _pointer(status), stream_ptr()))
    return out, offsets, status


@_on_device
def rows_pwm_max(base, starts, lens, enc_mode, matrix, lut=None, status=None):
    """K7 fused with the row maximum: float64[R], NaN-propagating, -inf for a row without a window; the scores are
    never written.  Returns (max, status)."""
    (head, lut_p), pwm = _rows_args(base, starts, lens, lut, status=status), _pwm_args(matrix)
    out = torch.empty(lens.numel(), dtype=torch.float64, device=base.device)
    status = nv.new_status(base.device) if status is None else status
    check(lib().bnpk_rows_pwm_max(*head, enc_mode, lut_p, *pwm, _pointer(out), _pointer(status), stream_ptr()))
    return out, status


def _match_args(alphabet_size, sets, sub_lens):
    """sets: int32 (uint32 words) on the device; sub_lens: a host sequence of ints."""
    lens = (ctypes.c_int32 * len(sub_lens))(*[int(x) for x in sub_lens])
    return alphabet_size, _pointer(sets, "sets", torch.int32), ctypes.cast(lens, ctypes.c_void_p), len(sub_lens)


@_on_device
def rows_match(base, starts, lens, enc_mode, alphabet_size, sets, sub_lens, same=False, lut=None, offsets=None,
               status=None, total=None, out=None):
    """K8: 1 where some sub-pattern matches at a position and fits in its row, else 0 (uint8): the windows of the
    longest sub-pattern, or every position with ``same``.  ``out`` (uint8[total], written at ``offsets``) is written in
    place when given.  Returns (matches, offsets, status)."""
    head, lut_p = _rows_args(base, starts, lens, lut, offsets, status)
    match = _match_args(alphabet_size, sets, sub_lens)
    _pointer(out, "out", torch.uint8, at_least=total or 0, optional=True)
    if out is None:
        span = max(map(int, sub_lens), default=1)
        out, offsets = _ragged_out(lens, 0 if same else span - 1, offsets, total, torch.uint8)
    elif offsets is None:
        raise ValueError("rows_match writes a given out at the given offsets")
    status = nv.new_status(base.device) if status is None else status
    check(lib().bnpk_rows_match(*head, enc_mode, lut_p, *match, int(same), _pointer(offsets), _pointer(out),
                                _pointer(status), stream_ptr()))
    return out, offsets, status


@_on_device
def rows_match_count(base, starts, lens, enc_mode, alphabet_size, sets, sub_lens, same=False, lut=None, status=None):
    """K8 fused with the row sum: int64[R] matches per row; the matches are never written.  Returns (counts, status)."""
    head, lut_p = _rows_args(base, starts, lens, lut, status=status)
    match = _match_args(alphabet_size, sets, sub_lens)
    out = torch.empty(lens.numel(), dtype=torch.int64, device=base.device)
    status = nv.new_status(base.device) if status is None else status
    check(lib().bnpk_rows_match_count(*head, enc_mode, lut_p, *match, int(same), _pointer(out), _pointer(status),
                                      stream_ptr()))
    return out, status


@_on_device
def bincount(values, n_bins, hist=None, hist_mode=nv.HIST_AUTO, status=None):
    values_p, _ = _pointer(values, "values", torch.int64), _status(status)
    hist = _hist(hist, n_bins, values.device)
    status = nv.new_status(values.device) if status is None else status
    check(lib().bnpk_bincount(values_p, values.numel(), n_bins, hist_mode, _pointer(hist), _pointer(status),
                              stream_ptr()))
    return hist, status


@_on_device
def bincount_rows(values, offsets, n_bins, status=None):
    values_p, offsets_p, _ = (_pointer(values, "values", torch.int64),
                              _pointer(offsets, "offsets", torch.int64, at_least=1), _status(status))
    n_rows = offsets.numel() - 1
    out = torch.zeros((n_rows, n_bins), dtype=torch.int64, device=values.device)
    status = nv.new_status(values.device) if status is None else status
    check(lib().bnpk_bincount_rows(values_p, offsets_p, n_rows, n_bins, _pointer(out), _pointer(status), stream_ptr()))
    return out, status


@_on_device
def synth_fastq(n_records, first_record=0, seed=20240924, device="cuda", out=None):
    """Synthetic 317-byte FASTQ records on the device (bit-identical to the oracle's generator)."""
    if out is None:
        out = torch.empty(n_records * 317, dtype=torch.uint8, device=device)
        return synth_fastq(n_records, first_record, seed, out=out)
    check(lib().bnpk_synth_fastq(_pointer(out, "out", torch.uint8, at_least=n_records * 317), first_record, n_records,
                                 seed, stream_ptr()))
    return out


class HostPipeline:
    """bnpk_pipeline_*: host chunk -> sliced H2D overlapped with the fused count."""

    def __init__(self, capacity_bytes, slice_bytes=64 << 20):
        self._h = ctypes.c_void_p(0)
        check(lib().bnpk_pipeline_create(ctypes.byref(self._h), capacity_bytes, slice_bytes))
        self.capacity = capacity_bytes

    @_on_device
    def kmer_count(self, chunk_host, k, hist, window_size=0, lines_per_entry=4, header_char=ord("@"),
                   check_plus=True, trim_cr=-1, enc_mode=nv.ENC_ASCII_ACGT, lut_host=None, hist_mode=nv.HIST_AUTO):
        """chunk_host: host uint8 tensor (pinned for real overlap); lut_host: host uint8[256] or None; hist: CUDA
        int64[n_bins], whose device runs the count."""
        status = (ctypes.c_int64 * nv.ST_WORDS)()
        check(lib().bnpk_pipeline_kmer_count_host_on(
            self._h, _pointer(chunk_host, "chunk_host", torch.uint8, host=True), chunk_host.numel(), lines_per_entry,
            header_char, int(check_plus), trim_cr, enc_mode,
            _pointer(lut_host, "lut_host", torch.uint8, n=256, optional=True, host=True), k, window_size,
            hist.numel(), hist_mode, _pointer(hist, "hist", torch.int64), ctypes.cast(status, ctypes.c_void_p),
            stream_ptr()))
        return ScanStatus(list(status))

    def close(self):
        if self._h:
            nv.load_library().bnpk_pipeline_destroy(self._h)
            self._h = ctypes.c_void_p(0)

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


@_on_device
def multiline_flags(chunk, starts, lens):
    """bnpk_multiline_flags over the lines (starts, lens) of ``chunk``: (is_header int32, out2 int64[2] = 1 + the last
    line whose newline is followed by '>' (0: no complete entry), 1 if one of the first ten lines ends in '\\r')."""
    head, _ = _rows_args(chunk, starts, lens)
    is_header = torch.empty(lens.numel(), dtype=torch.int32, device=chunk.device)
    out2 = torch.zeros(2, dtype=torch.int64, device=chunk.device)
    check(lib().bnpk_multiline_flags(*head, _pointer(is_header), _pointer(out2), stream_ptr()))
    return is_header, out2


@_on_device
def multiline_entries(chunk, starts, lens, is_header, hdr_before, n_entries, trim_cr):
    """bnpk_multiline_entries with hdr_before = row_offsets(is_header) and its total ``n_entries``: every entry's header
    (h_starts, h_lens), the sequence lines in order (s_starts, s_lens) and the bases of every entry (entry_lens)."""
    (chunk_p, _, starts_p, lens_p, n), _ = _rows_args(chunk, starts, lens)
    flags_p = _pointer(is_header, "is_header", torch.int32, n=n)
    before_p = _pointer(hdr_before, "hdr_before", torch.int64, at_least=n + 1)
    dev = chunk.device
    h_starts, s_starts = (torch.empty(m, dtype=torch.int64, device=dev) for m in (n_entries, n - n_entries))
    h_lens, s_lens = (torch.empty(m, dtype=torch.int32, device=dev) for m in (n_entries, n - n_entries))
    entry_lens = torch.zeros(n_entries, dtype=torch.int64, device=dev)
    check(lib().bnpk_multiline_entries(chunk_p, starts_p, lens_p, flags_p, before_p, n, int(trim_cr),
                                       _pointer(h_starts), _pointer(h_lens), _pointer(s_starts), _pointer(s_lens),
                                       _pointer(entry_lens), stream_ptr()))
    return h_starts, h_lens, s_starts, s_lens, entry_lens


@_on_device
def bloom_insert(values, hash_offsets, mask):
    """bnpk_bloom_insert: uint8 mask[(v ^ hash_offsets[i]) % mask size] = 1 for every value v and function i (int64)."""
    check(lib().bnpk_bloom_insert(_pointer(values, "values", torch.int64), values.numel(),
                                  _pointer(hash_offsets, "hash_offsets", torch.int64), hash_offsets.numel(),
                                  _pointer(mask, "mask", torch.uint8), mask.numel(), stream_ptr()))


@_on_device
def bloom_query(values, hash_offsets, mask):
    """bnpk_bloom_query: uint8[V], 1 where the mask holds every hash function's position of the value."""
    values_p = _pointer(values, "values", torch.int64)
    offsets_p, mask_p = _pointer(hash_offsets, "hash_offsets", torch.int64), _pointer(mask, "mask", torch.uint8)
    out = torch.empty(values.numel(), dtype=torch.uint8, device=mask.device)
    check(lib().bnpk_bloom_query(values_p, values.numel(), offsets_p, hash_offsets.numel(), mask_p, mask.numel(),
                                 _pointer(out), stream_ptr()))
    return out


def _text_out(offsets, out_begin, out_end, out):
    """(out_end, out): out_end defaults to offsets[-1] (read back), out holds the uint8 bytes [out_begin, out_end)."""
    if out_end is None:
        out_end = int(offsets[-1].item())
    size = max(out_end - out_begin, 0)
    _pointer(out, "out", torch.uint8, at_least=size, optional=True)
    return out_end, torch.empty(size, dtype=torch.uint8, device=offsets.device) if out is None else out


def _format_fields(fields):
    """A host bnpk_field[3] of (name, sequence, quality); each a (base uint8, starts int64, lens int32, lut uint8[256]
    or None) of CUDA tensors, or None.  Returns (array, number of entries, device)."""
    arr = (nv.Field * 3)()
    n, dev = None, None
    for i, f in enumerate(fields):
        if f is None:
            continue
        (base_p, base_bytes, starts_p, lens_p, rows), lut_p = _rows_args(*f)
        if n is None:
            n, dev = rows, f[0].device
        if rows != n:
            raise ValueError("every field needs one row per entry")
        arr[i] = nv.Field(base_p.value, base_bytes, starts_p.value, lens_p.value, lut_p.value)
    return arr, n or 0, dev


@_on_device
def format_offsets(fmt, line_width, fields, status=None):
    """int64[E+1] output offsets of the records (name, sequence, quality fields) in format ``fmt`` (nv.FMT_*) and the
    status tensor; with a sequence LUT, a sequence byte the LUT maps to 0 is reported in status[ST_BAD_BASE]."""
    arr, n, dev = _format_fields(fields)
    if dev is None:
        raise ValueError("format_offsets needs the name and sequence fields")
    _status(status)
    offsets = torch.empty(n + 1, dtype=torch.int64, device=dev)
    status = nv.new_status(dev) if status is None else status
    ws = nv.workspace(max(n, 1), dev)
    check(lib().bnpk_format_offsets(fmt, line_width, n, ctypes.cast(arr, ctypes.c_void_p), _pointer(offsets),
                                    _pointer(status), _pointer(ws), ws.numel(), stream_ptr()))
    return offsets, status


@_on_device
def format_records(fmt, line_width, fields, offsets, out_begin=0, out_end=None, out=None):
    """Bytes [out_begin, out_end) of the formatted records (default: all of them, offsets[-1] read back) into ``out``
    (uint8, at least out_end - out_begin bytes; allocated when None).  Returns ``out``."""
    arr, n, _ = _format_fields(fields)
    offsets_p = _pointer(offsets, "offsets", torch.int64, at_least=n + 1)
    out_end, out = _text_out(offsets, out_begin, out_end, out)
    check(lib().bnpk_format_records(fmt, line_width, n, ctypes.cast(arr, ctypes.c_void_p), offsets_p, out_begin,
                                    out_end, _pointer(out), stream_ptr()))
    return out


@_on_device
def delimited_columns(chunk, starts, lens, kinds, status=None):
    """The tab-separated columns of the lines (starts, lens) of ``chunk``, one nv.COL_* kind per column.  Returns
    (columns, status): per column None (COL_SKIP), (starts int64, lens int32) of text, int64 values or uint8 strand
    codes; the first fault is (line << 8 | column << 3 | nv.BAD_*) in status[ST_BAD_BASE]."""
    head, _ = _rows_args(chunk, starts, lens, status=status)
    n, dev = lens.numel(), chunk.device
    if not 1 <= len(kinds) <= nv.MAX_COLUMNS:
        raise ValueError(f"1 to {nv.MAX_COLUMNS} columns")
    arr = (nv.Column * len(kinds))()
    cols = []
    for i, kind in enumerate(kinds):
        if kind == nv.COL_TEXT:
            col = (torch.empty(n, dtype=torch.int64, device=dev), torch.empty(n, dtype=torch.int32, device=dev))
            arr[i] = nv.Column(kind, _pointer(col[0]).value, _pointer(col[1]).value)
        elif kind in (nv.COL_INT, nv.COL_INT_OR_DOT, nv.COL_STRAND):
            col = torch.empty(n, dtype=torch.uint8 if kind == nv.COL_STRAND else torch.int64, device=dev)
            arr[i] = nv.Column(kind, _pointer(col).value, None)
        else:
            col = None
            arr[i] = nv.Column(kind, None, None)
        cols.append(col)
    status = nv.new_status(dev) if status is None else status
    check(lib().bnpk_delimited_columns(*head, ctypes.cast(arr, ctypes.c_void_p), len(kinds), _pointer(status),
                                       stream_ptr()))
    return cols, status


@_on_device
def name_lookup(base, starts, lens, names, name_offsets, status=None):
    """The index of each row's bytes in the sorted name table (names uint8, name_offsets int64[C+1]): int32, -1 for an
    unknown name, whose row is reported in status[ST_BAD_BASE].  Returns (ids, status)."""
    head, _ = _rows_args(base, starts, lens, status=status)
    names_p = _pointer(names, "names", torch.uint8)
    name_offsets_p = _pointer(name_offsets, "name_offsets", torch.int64, at_least=1)
    ids = torch.empty(lens.numel(), dtype=torch.int32, device=base.device)
    status = nv.new_status(base.device) if status is None else status
    check(lib().bnpk_name_lookup(*head, names_p, name_offsets_p, name_offsets.numel() - 1, _pointer(ids),
                                 _pointer(status), stream_ptr()))
    return ids, status


def _intervals(start, stop):
    """(start, stop, R) of R intervals: int64 starts and one int64 stop per start."""
    start_p = _pointer(start, "start", torch.int64)
    return start_p, _pointer(stop, "stop", torch.int64, n=start.numel()), start.numel()


def _interval_args(file, start, stop, ids, contigs):
    """The head of a bnpk_interval_gather call: the file (uint8), the intervals and, with ``ids`` (int32, one per
    interval), the contig columns (offset int64, lenc int32, lenb int32, length int64) of one length."""
    file_p, (start_p, stop_p, n) = _pointer(file, "file", torch.uint8), _intervals(start, stop)
    if ids is None:
        return [file_p, file.numel(), n, None, None, None, None, None, 0, start_p, stop_p]
    offset, lenc, lenb, length = contigs
    offset_p, c = _pointer(offset, "contig_offset", torch.int64), offset.numel()
    return [file_p, file.numel(), n, _pointer(ids, "ids", torch.int32, n=n), offset_p,
            _pointer(lenc, "lenc", torch.int32, n=c), _pointer(lenb, "lenb", torch.int32, n=c),
            _pointer(length, "contig_len", torch.int64, n=c), c, start_p, stop_p]


@_on_device
def interval_check(file, start, stop, ids=None, contigs=None, status=None):
    """The check pass of bnpk_interval_gather: (row_lens int32 = stop - start, 0 for a bad row; status with the first
    bad row in ST_BAD_BASE).  ``contigs`` = (offset int64, lenc int32, lenb int32, length int64) indexed by ``ids``
    (int32); without ids the file is one contig without line ends."""
    args, _ = _interval_args(file, start, stop, ids, contigs), _status(status)
    row_lens = torch.empty(start.numel(), dtype=torch.int32, device=file.device)
    status = nv.new_status(file.device) if status is None else status
    check(lib().bnpk_interval_gather(*args, None, None, _pointer(row_lens), None, None, _pointer(status),
                                     stream_ptr()))
    return row_lens, status


@_on_device
def interval_copy(file, start, stop, offsets, total, ids=None, contigs=None, strand=None, complement_lut=None):
    """The copy pass: uint8[total], row r at offsets[r] (int64[R+1] of interval_check's row_lens), a row whose
    strand[r] (uint8) is not 0 reverse-complemented through ``complement_lut`` (uint8[256])."""
    args = _interval_args(file, start, stop, ids, contigs)
    offsets_p = _pointer(offsets, "offsets", torch.int64, n=start.numel() + 1)
    strand_p = _pointer(strand, "strand", torch.uint8, n=start.numel(), optional=True)
    lut_p = _pointer(complement_lut, "complement_lut", torch.uint8, n=256, optional=strand is None)
    out = torch.empty(total, dtype=torch.uint8, device=file.device)
    if total:
        check(lib().bnpk_interval_gather(*args, strand_p, lut_p, None, offsets_p, _pointer(out), None, stream_ptr()))
    return out


def interval_gather(file, start, stop, ids=None, contigs=None, strand=None, complement_lut=None, extra=()):
    """Both passes of bnpk_interval_gather around the one synchronisation a gather needs: the check pass, the row
    offsets, then a single .cpu() of the output size, the first bad row and the ``extra`` one-word device tensors (a
    caller's own status words).  Returns (out, row_lens, bad_row, extra words).  With a bad row the copy pass is not
    launched and ``out`` is None: the caller words the error.  A row of more than INT32_MAX bases is a bad row."""
    row_lens, status = interval_check(file, start, stop, ids, contigs)
    offsets = row_offsets(row_lens)
    total, bad, *words = torch.cat([offsets[-1:], status[nv.ST_BAD_BASE:nv.ST_BAD_BASE + 1], *extra]).cpu().tolist()
    if bad != nv.INT64_MAX:
        return None, row_lens, bad, words
    return interval_copy(file, start, stop, offsets, total, ids, contigs, strand, complement_lut), row_lens, None, words


@_on_device
def interval_events(start, stop, ids=None, contig_offset=None, contig_len=None, size=0, keys=True, glob=False,
                    status=None):
    """bnpk_interval_events: (keys int64[2R] or None, global start, global stop (or None), status).  ``ids`` (int32)
    index contig_offset / contig_len (int64; an offset < 0 leaves the contig out); without ids every row is on one
    contig of ``size``.  A bad row is reported in status[ST_BAD_BASE]."""
    start_p, stop_p, n = _intervals(start, stop)
    contig = [None, None, None, 0]
    if ids is not None:
        ids_p, offset_p = _pointer(ids, "ids", torch.int32, n=n), _pointer(contig_offset, "contig_offset", torch.int64)
        contig = [ids_p, offset_p, _pointer(contig_len, "contig_len", torch.int64, n=contig_offset.numel()),
                  contig_offset.numel()]
    _status(status)
    dev = start.device
    k = torch.empty(2 * n, dtype=torch.int64, device=dev) if keys else None
    gs, ge = (torch.empty(n, dtype=torch.int64, device=dev) for _ in range(2)) if glob else (None, None)
    status = nv.new_status(dev) if status is None else status
    check(lib().bnpk_interval_events(start_p, stop_p, *contig, size, n, _pointer(k, optional=True),
                                     _pointer(gs, optional=True), _pointer(ge, optional=True), _pointer(status),
                                     stream_ptr()))
    return k, gs, ge, status


@_on_device
def pileup_runs(sorted_keys, size, mode=nv.PILEUP_COUNT):
    """bnpk_pileup_runs on sorted event keys: (run_starts int64[K + 2], run_values int64[K + 1], n_runs int64[1]), the
    first n_runs + 1 starts and n_runs values valid (nothing is read back)."""
    keys_p = _pointer(sorted_keys, "keys", torch.int64)
    n, dev = sorted_keys.numel(), sorted_keys.device
    starts = torch.empty(n + 2, dtype=torch.int64, device=dev)
    values = torch.empty(n + 1, dtype=torch.int64, device=dev)
    n_runs = torch.empty(1, dtype=torch.int64, device=dev)
    ws = nv.workspace(max(n, 1), dev)
    check(lib().bnpk_pileup_runs(keys_p, n, size, mode, _pointer(starts), _pointer(values), _pointer(n_runs),
                                 _pointer(ws), ws.numel(), stream_ptr()))
    return starts, values, n_runs


def _runs_args(run_starts, values, min_runs=0):
    """(run_starts, values, R) of a track: R int64 values (at least ``min_runs``) and R + 1 int64 run starts."""
    values_p = _pointer(values, "values", torch.int64, at_least=min_runs)
    return _pointer(run_starts, "run_starts", torch.int64, n=values.numel() + 1), values_p, values.numel()


@_on_device
def runs_reduce(run_starts, values, q_start, q_stop, mode):
    """bnpk_runs_reduce: int64[Q], one reduction (nv.RUNS_*) per query [q_start, q_stop); no synchronisation."""
    runs, (q0_p, q1_p, n) = _runs_args(run_starts, values, 1), _intervals(q_start, q_stop)
    dev = q_start.device
    out = torch.empty(n, dtype=torch.int64, device=dev)
    scratch = torch.empty(3 * n + 1, dtype=torch.int64, device=dev)
    ws = nv.workspace(max(n, 1), dev)
    check(lib().bnpk_runs_reduce(*runs, q0_p, q1_p, n, mode, _pointer(out), _pointer(scratch), _pointer(ws),
                                 ws.numel(), stream_ptr()))
    return out


@_on_device
def runs_extract(run_starts, values, q_start, out_offsets, total):
    """bnpk_runs_extract: int64[total], query q's values at out_offsets[q] (int64[Q + 1])."""
    runs, q_p = _runs_args(run_starts, values, 1), _pointer(q_start, "q_start", torch.int64)
    offsets_p = _pointer(out_offsets, "out_offsets", torch.int64, n=q_start.numel() + 1)
    out = torch.empty(total, dtype=torch.int64, device=q_start.device)
    if total:
        check(lib().bnpk_runs_extract(*runs, q_p, q_start.numel(), offsets_p, _pointer(out), stream_ptr()))
    return out


@_on_device
def interval_merge(start, stop, same_prev=None, distance=0, status=None):
    """bnpk_interval_merge: (out_rows int64[R], out_stops int64[R], n_out int64[1], status), the first n_out entries
    valid; a start that decreases inside a segment is reported in status[ST_BAD_BASE]."""
    start_p, stop_p, n = _intervals(start, stop)
    same_p, _ = _pointer(same_prev, "same_prev", torch.uint8, n=n, optional=True), _status(status)
    dev = start.device
    rows, stops = (torch.empty(n, dtype=torch.int64, device=dev) for _ in range(2))
    n_out = torch.empty(1, dtype=torch.int64, device=dev)
    status = nv.new_status(dev) if status is None else status
    ws = nv.workspace(max(n, 1), dev)
    check(lib().bnpk_interval_merge(start_p, stop_p, same_p, n, max(int(distance), 0), _pointer(rows), _pointer(stops),
                                    _pointer(n_out), _pointer(status), _pointer(ws), ws.numel(), stream_ptr()))
    return rows, stops, n_out, status


@_on_device
def rows_equal_prev(base, starts, lens):
    """bnpk_rows_equal_prev: uint8[R], 1 where a row's bytes equal the previous row's."""
    head, _ = _rows_args(base, starts, lens)
    flag = torch.empty(lens.numel(), dtype=torch.uint8, device=base.device)
    check(lib().bnpk_rows_equal_prev(*head, _pointer(flag), stream_ptr()))
    return flag


@_on_device
def runs_combine(a_starts, a_values, b_starts, b_values, op):
    """bnpk_runs_combine: (run_starts int64[Ra + Rb + 1], run_values int64[Ra + Rb], n_runs int64[1]), the canonical
    runs of op(A, B) (nv.OP_*) of two tracks of one size, the first n_runs + 1 starts and n_runs values valid (nothing
    is read back)."""
    a, b = _runs_args(a_starts, a_values), _runs_args(b_starts, b_values)
    n, dev = a[2] + b[2], a_starts.device
    starts = torch.empty(n + 1, dtype=torch.int64, device=dev)
    values = torch.empty(max(n, 1), dtype=torch.int64, device=dev)
    n_runs = torch.empty(1, dtype=torch.int64, device=dev)
    ws = nv.workspace(max(n, 1), dev)
    check(lib().bnpk_runs_combine(*a, *b, op, _pointer(starts), _pointer(values), _pointer(n_runs), _pointer(ws),
                                  ws.numel(), stream_ptr()))
    return starts, values, n_runs


@_on_device
def interval_intersect(start, stop, same_prev=None, rows=True):
    """bnpk_interval_intersect over rows sorted by start and, separately, their stops sorted (inside each segment of
    ``same_prev``, uint8): (out_rows int64[R] or None, out_stops int64[R] or None, n_out int64[1], overlap int64[1]),
    the first n_out rows valid.  ``rows=False`` counts the pairs and sums their overlaps only."""
    start_p, stop_p, n = _intervals(start, stop)
    same_p = _pointer(same_prev, "same_prev", torch.uint8, n=n, optional=True)
    dev = start.device
    out_rows, out_stops = (torch.empty(n, dtype=torch.int64, device=dev) for _ in range(2)) if rows else (None, None)
    n_out, overlap = (torch.empty(1, dtype=torch.int64, device=dev) for _ in range(2))
    ws = nv.workspace(max(n, 1), dev)
    check(lib().bnpk_interval_intersect(start_p, stop_p, same_p, n, _pointer(out_rows, optional=True),
                                        _pointer(out_stops, optional=True), _pointer(n_out), _pointer(overlap),
                                        _pointer(ws), ws.numel(), stream_ptr()))
    return out_rows, out_stops, n_out, overlap


@_on_device
def runs_to_intervals(run_starts, values, contig_ends, mode=nv.RUNS_TO_NONZERO):
    """bnpk_runs_to_intervals: the rows of a global track cut at the contig ends (int64[C + 1], strictly increasing
    from 0 to the size): (contig int32, start int64, stop int64, value int64 or None, n_out int64[1]), each of capacity
    R + C, the first n_out rows valid (nothing is read back).  nv.RUNS_TO_NONZERO: the stretches of non-zero value;
    nv.RUNS_TO_ALL: every run, with its value."""
    runs, ends_p = _runs_args(run_starts, values), _pointer(contig_ends, "contig_ends", torch.int64, at_least=2)
    n, c, dev = values.numel(), contig_ends.numel() - 1, run_starts.device
    contig = torch.empty(n + c, dtype=torch.int32, device=dev)
    start, stop = (torch.empty(n + c, dtype=torch.int64, device=dev) for _ in range(2))
    value = torch.empty(n + c, dtype=torch.int64, device=dev) if mode == nv.RUNS_TO_ALL else None
    n_out = torch.empty(1, dtype=torch.int64, device=dev)
    ws = nv.workspace(max(n, 1), dev)
    check(lib().bnpk_runs_to_intervals(*runs, ends_p, c, mode, _pointer(contig), _pointer(start), _pointer(stop),
                                       _pointer(value, optional=True), _pointer(n_out), _pointer(ws), ws.numel(),
                                       stream_ptr()))
    return contig, start, stop, value, n_out


def _out_columns(columns):
    """A host bnpk_out_column[k] of columns given as (nv.COL_TEXT, (base uint8, starts int64, lens int32)),
    (nv.COL_INT, int64) or (nv.COL_STRAND, uint8) CUDA tensors of one row count.  Returns (array, rows, device)."""
    if not 1 <= len(columns) <= nv.MAX_OUT_COLUMNS:
        raise ValueError(f"1 to {nv.MAX_OUT_COLUMNS} columns")
    arr = (nv.OutColumn * len(columns))()
    rows, dev = None, None
    for i, (kind, data) in enumerate(columns):
        if kind == nv.COL_TEXT:
            (base_p, base_bytes, starts_p, lens_p, n), _ = _rows_args(*data)
            arr[i] = nv.OutColumn(kind, base_p.value, base_bytes, starts_p.value, lens_p.value)
            d = data[0].device
        elif kind in (nv.COL_INT, nv.COL_STRAND):
            data_p = _pointer(data, "column", torch.int64 if kind == nv.COL_INT else torch.uint8)
            arr[i] = nv.OutColumn(kind, data_p.value, 0, None, None)
            n, d = data.numel(), data.device
        else:
            raise ValueError(f"unknown column kind {kind}")
        if rows is None:
            rows, dev = n, d
        if n != rows:
            raise ValueError(f"the columns differ in length ({rows} and {n} rows)")
    return arr, rows, dev


@_on_device
def delimited_offsets(columns, status=None):
    """bnpk_delimited_offsets: (int64[E + 1] line offsets, status); a strand code above 2 is reported in
    status[ST_BAD_BASE] as (line << 8 | column << 3 | nv.BAD_STRAND)."""
    arr, n, dev = _out_columns(columns)
    _status(status)
    offsets = torch.empty(n + 1, dtype=torch.int64, device=dev)
    status = nv.new_status(dev) if status is None else status
    ws = nv.workspace(max(n, 1), dev)
    check(lib().bnpk_delimited_offsets(ctypes.cast(arr, ctypes.c_void_p), len(columns), n, _pointer(offsets),
                                       _pointer(status), _pointer(ws), ws.numel(), stream_ptr()))
    return offsets, status


@_on_device
def delimited_format(columns, offsets, out_begin=0, out_end=None, out=None):
    """Bytes [out_begin, out_end) of the lines (default: all, offsets[-1] read back) into ``out`` (uint8, at least
    out_end - out_begin bytes; allocated when None).  Returns ``out``."""
    arr, n, _ = _out_columns(columns)
    offsets_p = _pointer(offsets, "offsets", torch.int64, n=n + 1)
    out_end, out = _text_out(offsets, out_begin, out_end, out)
    check(lib().bnpk_delimited_format(ctypes.cast(arr, ctypes.c_void_p), len(columns), n, offsets_p, out_begin,
                                      out_end, _pointer(out), stream_ptr()))
    return out


BAM_SEGMENT_BYTES = 4096        # the bytes one warp of the BAM split speculates on (DESIGN §3 K15)
BAM_MIN_RECORD = 36             # block_size word + the 32 fixed bytes


@_on_device
def bam_split(chunk, n_ref, segment_bytes=BAM_SEGMENT_BYTES, status=None):
    """bnpk_bam_split: (starts int64[n // 36 + 1], status).  The first status[ST_N_RECORDS] starts are the chunk's
    complete records; status[ST_N_COMPLETE_BYTES] is their size, status[ST_BAD_BASE] the first fault as
    (record << 8 | nv.BAM_BAD_*) and status[ST_N_VALUES] the number of segments walked again."""
    chunk_p = _pointer(chunk, "chunk", torch.uint8)
    _status(status)
    if segment_bytes < 64:
        raise ValueError("segment_bytes must be at least 64")
    n, dev = chunk.numel(), chunk.device
    starts = torch.empty(n // BAM_MIN_RECORD + 1, dtype=torch.int64, device=dev)
    status = nv.new_status(dev) if status is None else status
    ws = torch.empty(7 * max(-(-n // segment_bytes), 1), dtype=torch.int64, device=dev)
    check(lib().bnpk_bam_split(chunk_p, n, n_ref, segment_bytes, _pointer(starts), starts.numel(), _pointer(status),
                               _pointer(ws), ws.numel(), stream_ptr()))
    return starts, status


@_on_device
def bam_fields(chunk, starts, status):
    """bnpk_bam_fields: int64[BAM_FIELDS, R] (R = starts.numel()); column r < status[ST_N_RECORDS] holds record r's
    fields (nv.BAM_F_*).  A cigar op code above 8 is reported in status[ST_BAD_BASE]."""
    chunk_p, starts_p = _pointer(chunk, "chunk", torch.uint8), _pointer(starts, "starts", torch.int64)
    status_p = _status(status, optional=False)
    fields = torch.empty(nv.BAM_FIELDS, starts.numel(), dtype=torch.int64, device=chunk.device)
    check(lib().bnpk_bam_fields(chunk_p, chunk.numel(), starts_p, starts.numel(), _pointer(fields), status_p,
                                stream_ptr()))
    return fields


@_on_device
def bam_sequence(chunk, seq_start, offsets, total):
    """bnpk_bam_sequence: uint8[total], the 4-bit base codes of the rows at offsets[r] .. offsets[r + 1]."""
    chunk_p, start_p = _pointer(chunk, "chunk", torch.uint8), _pointer(seq_start, "seq_start", torch.int64)
    offsets_p = _pointer(offsets, "offsets", torch.int64, n=seq_start.numel() + 1)
    out = torch.empty(total, dtype=torch.uint8, device=chunk.device)
    if total == 0:
        return out
    check(lib().bnpk_bam_sequence(chunk_p, chunk.numel(), start_p, offsets_p, seq_start.numel(), _pointer(out),
                                  stream_ptr()))
    return out


@_on_device
def bam_cigar(chunk, cigar_start, offsets, total):
    """bnpk_bam_cigar: (op uint8[total], length int64[total]) of the rows' cigar words at offsets[r] .. offsets[r + 1]."""
    chunk_p, start_p = _pointer(chunk, "chunk", torch.uint8), _pointer(cigar_start, "cigar_start", torch.int64)
    offsets_p = _pointer(offsets, "offsets", torch.int64, n=cigar_start.numel() + 1)
    op = torch.empty(total, dtype=torch.uint8, device=chunk.device)
    length = torch.empty(total, dtype=torch.int64, device=chunk.device)
    if total == 0:
        return op, length
    check(lib().bnpk_bam_cigar(chunk_p, chunk.numel(), start_p, offsets_p, cigar_start.numel(), _pointer(op),
                               _pointer(length), stream_ptr()))
    return op, length
