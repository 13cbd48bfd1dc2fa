"""Tensor-level wrappers over the C-ABI (include/bnpk.h).  Everything here runs on the current
CUDA stream of the current device; tensors must be contiguous CUDA tensors.  These are the
operator-level mirror of the reference functions named in include/bnpk.h."""
import ctypes

import torch

from . import _native as nv
from ._native import check, lib, ptr, stream_ptr


def _need_cuda(t, name="tensor"):
    if not isinstance(t, torch.Tensor) or not t.is_cuda:
        raise nv.NativeLibraryError(f"{name} must be a CUDA tensor: bionumpy_b200 has no CPU fallback")
    if not t.is_contiguous():
        raise ValueError(f"{name} must be contiguous")


def _on_device(fn):
    """Run an op with the device of its first tensor argument current (kernels launch on the current device's
    current stream) and check that every tensor argument lives there."""
    import functools

    @functools.wraps(fn)
    def wrapper(*args, **kwargs):
        tensors = [x for x in list(args) + list(kwargs.values()) if isinstance(x, torch.Tensor)]
        dev = next((t.device for t in tensors if t.is_cuda), None)
        if dev is None:
            return fn(*args, **kwargs)
        for t in tensors:
            if t.is_cuda and t.device != dev:
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
def count_byte(chunk, value: int) -> int:
    _need_cuda(chunk, "chunk")
    out = torch.empty(1, dtype=torch.int64, device=chunk.device)
    check(lib().bnpk_count_byte(ptr(chunk), chunk.numel(), value, ptr(out), stream_ptr()))
    return int(out.item())


@_on_device
def line_split(chunk, lines_per_entry=4, field_line=1, start_offset=0, header_char=ord("@"), check_plus=True,
               trim_cr=-1, max_rows=None):
    """K1.  Returns (starts int64[R'], lens int32[R'], status tensor).  R' = max_rows (default: the
    exact number of lines / lines_per_entry, obtained with one census pass)."""
    _need_cuda(chunk, "chunk")
    n = chunk.numel()
    dev = chunk.device
    if max_rows is None:
        max_rows = count_byte(chunk, 10) // lines_per_entry
    starts = torch.empty(max_rows, dtype=torch.int64, device=dev)
    lens = torch.empty(max_rows, dtype=torch.int32, device=dev)
    status = nv.new_status(dev)
    ws = nv.workspace(n, dev)
    check(lib().bnpk_line_split(ptr(chunk), n, lines_per_entry, field_line, start_offset, header_char,
                                int(check_plus), trim_cr, ptr(starts), ptr(lens), max_rows, ptr(status),
                                ptr(ws), ws.numel(), stream_ptr()))
    return starts, lens, status


@_on_device
def chunk_kmer_count(chunk, k, n_bins, hist=None, window_size=0, lines_per_entry=4, header_char=ord("@"),
                     check_plus=True, trim_cr=-1, enc_mode=nv.ENC_ASCII_ACGT, lut=None, hist_mode=nv.HIST_AUTO,
                     status=None):
    """K6 on a device-resident chunk.  Accumulates into ``hist`` (int64[n_bins]); returns
    (hist, status tensor)."""
    _need_cuda(chunk, "chunk")
    n = chunk.numel()
    dev = chunk.device
    if hist is None:
        hist = torch.zeros(n_bins, dtype=torch.int64, device=dev)
    if status is None:
        status = nv.new_status(dev)
    ws = nv.workspace(n, dev)
    check(lib().bnpk_chunk_kmer_count(ptr(chunk), n, 0, n, 1, lines_per_entry, header_char, int(check_plus),
                                      trim_cr, enc_mode, ptr(lut), k, window_size, n_bins, hist_mode, ptr(hist),
                                      ptr(status), ptr(ws), ws.numel(), stream_ptr()))
    return hist, status


@_on_device
def row_offsets(lens, shrink=0):
    """int64[R+1] exclusive prefix sums of max(lens - shrink, 0)."""
    _need_cuda(lens, "lens")
    if lens.dtype != torch.int32:
        raise TypeError("lens must be int32")
    n = lens.numel()
    out = torch.empty(n + 1, dtype=torch.int64, device=lens.device)
    ws = nv.workspace(max(n, 1), lens.device)
    check(lib().bnpk_row_offsets(ptr(lens), n, shrink, ptr(out), ptr(ws), ws.numel(), stream_ptr()))
    return out


def _ragged_out(lens, shrink, offsets, total, dtype):
    """The flat output of a row op and its row offsets: max(lens - shrink, 0) values per row unless ``offsets``
    (int64[R+1]) are given, ``total`` values (default offsets[-1])."""
    if offsets is None:
        offsets = row_offsets(lens, shrink)
    if total is None:
        total = int(offsets[-1].item())
    return torch.empty(total, dtype=dtype, device=lens.device), offsets


def _rows_args(base, starts, lens):
    _need_cuda(base, "base")
    _need_cuda(starts, "starts")
    _need_cuda(lens, "lens")
    if base.dtype != torch.uint8 or starts.dtype != torch.int64 or lens.dtype != torch.int32:
        raise TypeError("base must be uint8, starts int64, lens int32")
    if starts.numel() != lens.numel():
        raise ValueError("starts and lens differ in length")
    return ptr(base), base.numel(), ptr(starts), ptr(lens), lens.numel()


@_on_device
def rows_encode(base, starts, lens, enc_mode, lut=None, offsets=None, status=None, total=None):
    out, offsets = _ragged_out(lens, 0, offsets, total, torch.uint8)
    if status is None:
        status = nv.new_status(base.device)
    check(lib().bnpk_rows_encode(*_rows_args(base, starts, lens), enc_mode, ptr(lut), ptr(offsets), ptr(out),
                                 ptr(status), stream_ptr()))
    return out, offsets, status


@_on_device
def rows_kmer_hash(base, starts, lens, enc_mode, k, lut=None, offsets=None, status=None, total=None):
    out, offsets = _ragged_out(lens, k - 1, offsets, total, torch.int64)
    if status is None:
        status = nv.new_status(base.device)
    check(lib().bnpk_rows_kmer_hash(*_rows_args(base, starts, lens), enc_mode, ptr(lut), k, ptr(offsets), ptr(out),
                                    ptr(status), stream_ptr()))
    return out, offsets, status


@_on_device
def rows_generic_hash(base, starts, lens, alphabet_size, k, lut=None, offsets=None, status=None, total=None):
    """sum_j code[i+j] * alphabet_size^j for alphabets that are not four letters (K3')."""
    out, offsets = _ragged_out(lens, k - 1, offsets, total, torch.int64)
    if status is None:
        status = nv.new_status(base.device)
    check(lib().bnpk_rows_generic_hash(*_rows_args(base, starts, lens), ptr(lut), alphabet_size, k, ptr(offsets),
                                       ptr(out), ptr(status), stream_ptr()))
    return out, offsets, status


@_on_device
def rows_minimizers(base, starts, lens, enc_mode, k, window_size, lut=None, offsets=None, status=None, total=None):
    out, offsets = _ragged_out(lens, window_size - 1, offsets, total, torch.int64)
    if status is None:
        status = nv.new_status(base.device)
    check(lib().bnpk_rows_minimizers(*_rows_args(base, starts, lens), enc_mode, ptr(lut), k, window_size,
                                     ptr(offsets), ptr(out), ptr(status), stream_ptr()))
    return out, offsets, status


@_on_device
def rows_kmer_count(base, starts, lens, enc_mode, k, n_bins, window_size=0, lut=None, hist=None,
                    hist_mode=nv.HIST_AUTO, status=None):
    if hist is None:
        hist = torch.zeros(n_bins, dtype=torch.int64, device=base.device)
    if status is None:
        status = nv.new_status(base.device)
    check(lib().bnpk_rows_kmer_count(*_rows_args(base, starts, lens), enc_mode, ptr(lut), k, window_size, n_bins,
                                     hist_mode, ptr(hist), ptr(status), stream_ptr()))
    return hist, status


@_on_device
def rows_reverse_complement(base, starts, lens, lut, offsets=None, total=None):
    """get_reverse_complement on a ragged view: out row r = lut[row r backwards] (uint8, contiguous rows)."""
    out, offsets = _ragged_out(lens, 0, offsets, total, torch.uint8)
    check(lib().bnpk_rows_reverse_complement(*_rows_args(base, starts, lens), ptr(lut), ptr(offsets), ptr(out), stream_ptr()))
    return out, offsets


@_on_device
def rows_kmer_hash_canonical(base, starts, lens, enc_mode, k, complement_xor, lut=None, offsets=None, status=None,
                             total=None):
    """EXTENSION: min(h, hash of the reverse complement) for every k-mer (K3 with a second strand)."""
    out, offsets = _ragged_out(lens, k - 1, offsets, total, torch.int64)
    if status is None:
        status = nv.new_status(base.device)
    check(lib().bnpk_rows_kmer_hash_canonical(*_rows_args(base, starts, lens), enc_mode, ptr(lut), k, complement_xor,
                                              ptr(offsets), ptr(out), ptr(status), stream_ptr()))
    return out, offsets, status


@_on_device
def rows_kmer_count_canonical(base, starts, lens, enc_mode, k, complement_xor, n_bins, lut=None, hist=None,
                              hist_mode=nv.HIST_AUTO, status=None):
    if hist is None:
        hist = torch.zeros(n_bins, dtype=torch.int64, device=base.device)
    if status is None:
        status = nv.new_status(base.device)
    check(lib().bnpk_rows_kmer_count_canonical(*_rows_args(base, starts, lens), enc_mode, ptr(lut), k, complement_xor,
                                               n_bins, hist_mode, ptr(hist), ptr(status), stream_ptr()))
    return hist, status


def _table_args(keys, counts, n_used):
    for t, name in ((keys, "keys"), (counts, "counts"), (n_used, "n_used")):
        _need_cuda(t, name)
        if t.dtype != torch.int64:
            raise TypeError(f"{name} must be int64")
    if counts.numel() != keys.numel() or n_used.numel() != 1:
        raise ValueError("keys and counts must have the same length and n_used one element")
    return ptr(keys), ptr(counts), keys.numel(), ptr(n_used)


@_on_device
def rows_kmer_table_insert(base, starts, lens, enc_mode, k, keys, counts, n_used, complement_xor=0, lut=None,
                           status=None):
    """EXTENSION: insert every k-mer of the rows (canonical ones when complement_xor != 0) into the exact table
    (keys, counts: int64[C], C a power of two, free slot = key -1); n_used (int64[1]) grows by the slots claimed.
    Returns the status tensor."""
    if status is None:
        status = nv.new_status(base.device)
    check(lib().bnpk_rows_kmer_table_insert(*_rows_args(base, starts, lens), enc_mode, ptr(lut), k, complement_xor,
                                            *_table_args(keys, counts, n_used), ptr(status), stream_ptr()))
    return status


@_on_device
def kmer_table_rehash(keys, counts, new_keys, new_counts, n_used, status=None):
    """Re-insert every (key, count) of a table into a cleared one (growth); n_used grows by the slots claimed there."""
    if status is None:
        status = nv.new_status(keys.device)
    k_p, c_p, cap, _ = _table_args(keys, counts, n_used)
    nk_p, nc_p, new_cap, u_p = _table_args(new_keys, new_counts, n_used)
    check(lib().bnpk_kmer_table_rehash(k_p, c_p, cap, nk_p, nc_p, new_cap, u_p, ptr(status), stream_ptr()))
    return status


def _pwm_args(matrix, alphabet_size, lut):
    _need_cuda(matrix, "matrix")
    if matrix.dtype != torch.float64 or matrix.dim() != 2 or matrix.shape[1] != alphabet_size:
        raise TypeError("matrix must be float64 of shape [motif_len, alphabet_size]")
    if lut is not None:
        _need_cuda(lut, "lut")
    return ptr(lut), alphabet_size, ptr(matrix), matrix.shape[0]


@_on_device
def rows_pwm_scores(base, starts, lens, enc_mode, matrix, lut=None, tail=False, offsets=None, status=None, total=None):
    """K7: motif scores of every window of the rows (every position with ``tail``), float64, in column order.
    ``matrix`` is [motif_len, alphabet_size] on the device.  Returns (scores, offsets, status)."""
    alphabet_size = matrix.shape[-1] if matrix.dim() == 2 else 0
    out, offsets = _ragged_out(lens, 0 if tail else max(matrix.shape[0] - 1, 0), offsets, total, torch.float64)
    if status is None:
        status = nv.new_status(base.device)
    check(lib().bnpk_rows_pwm_scores(*_rows_args(base, starts, lens), enc_mode, *_pwm_args(matrix, alphabet_size, lut),
                                     int(tail), ptr(offsets), ptr(out), ptr(status), stream_ptr()))
    return out, offsets, status


@_on_device
def rows_pwm_max(base, starts, lens, enc_mode, matrix, lut=None, status=None):
    """K7 fused with the row maximum: float64[R], NaN-propagating, -inf for a row without a window; the scores are
    never written.  Returns (max, status)."""
    alphabet_size = matrix.shape[-1] if matrix.dim() == 2 else 0
    out = torch.empty(lens.numel(), dtype=torch.float64, device=base.device)
    if status is None:
        status = nv.new_status(base.device)
    check(lib().bnpk_rows_pwm_max(*_rows_args(base, starts, lens), enc_mode, *_pwm_args(matrix, alphabet_size, lut),
                                  ptr(out), ptr(status), stream_ptr()))
    return out, status


def _match_args(alphabet_size, sets, sub_lens, lut):
    """sets: int32 (uint32 words) on the device; sub_lens: a host sequence of ints."""
    _need_cuda(sets, "sets")
    if sets.dtype != torch.int32:
        raise TypeError("sets must be int32 words")
    if lut is not None:
        _need_cuda(lut, "lut")
    lens = (ctypes.c_int32 * len(sub_lens))(*[int(x) for x in sub_lens])
    return ptr(lut), alphabet_size, ptr(sets), ctypes.cast(lens, ctypes.c_void_p), len(sub_lens)


@_on_device
def rows_match(base, starts, lens, enc_mode, alphabet_size, sets, sub_lens, same=False, lut=None, offsets=None,
               status=None, total=None, out=None):
    """K8: 1 where some sub-pattern matches at a position and fits in its row, else 0 (uint8): the windows of the
    longest sub-pattern, or every position with ``same``.  ``out`` (uint8[total]) is written in place when given.
    Returns (matches, offsets, status)."""
    span = max(int(x) for x in sub_lens) if len(sub_lens) else 1
    if out is None:
        out, offsets = _ragged_out(lens, 0 if same else span - 1, offsets, total, torch.uint8)
    if status is None:
        status = nv.new_status(base.device)
    check(lib().bnpk_rows_match(*_rows_args(base, starts, lens), enc_mode, *_match_args(alphabet_size, sets, sub_lens, lut),
                                int(same), ptr(offsets), ptr(out), ptr(status), stream_ptr()))
    return out, offsets, status


@_on_device
def rows_match_count(base, starts, lens, enc_mode, alphabet_size, sets, sub_lens, same=False, lut=None, status=None):
    """K8 fused with the row sum: int64[R] matches per row; the matches are never written.  Returns (counts, status)."""
    out = torch.empty(lens.numel(), dtype=torch.int64, device=base.device)
    if status is None:
        status = nv.new_status(base.device)
    check(lib().bnpk_rows_match_count(*_rows_args(base, starts, lens), enc_mode,
                                      *_match_args(alphabet_size, sets, sub_lens, lut), int(same), ptr(out),
                                      ptr(status), stream_ptr()))
    return out, status


@_on_device
def bincount(values, n_bins, hist=None, hist_mode=nv.HIST_AUTO, status=None):
    _need_cuda(values, "values")
    if values.dtype != torch.int64:
        raise TypeError("values must be int64")
    if hist is None:
        hist = torch.zeros(n_bins, dtype=torch.int64, device=values.device)
    if status is None:
        status = nv.new_status(values.device)
    check(lib().bnpk_bincount(ptr(values), values.numel(), n_bins, hist_mode, ptr(hist), ptr(status), stream_ptr()))
    return hist, status


@_on_device
def bincount_rows(values, offsets, n_bins, status=None):
    _need_cuda(values, "values")
    n_rows = offsets.numel() - 1
    out = torch.zeros((n_rows, n_bins), dtype=torch.int64, device=values.device)
    if status is None:
        status = nv.new_status(values.device)
    check(lib().bnpk_bincount_rows(ptr(values), ptr(offsets), n_rows, n_bins, ptr(out), ptr(status), stream_ptr()))
    return out, status


def synth_fastq(n_records, first_record=0, seed=20240924, device="cuda", out=None):
    """Synthetic 317-byte FASTQ records on the device (bit-identical to the oracle's generator)."""
    if out is None:
        out = torch.empty(n_records * 317, dtype=torch.uint8, device=device)
    check(lib().bnpk_synth_fastq(ptr(out), first_record, n_records, seed, stream_ptr()))
    return out


class HostPipeline:
    """bnpk_pipeline_*: host chunk -> sliced H2D overlapped with the fused count."""

    def __init__(self, capacity_bytes, slice_bytes=64 << 20):
        self._h = ctypes.c_void_p(0)
        check(lib().bnpk_pipeline_create(ctypes.byref(self._h), capacity_bytes, slice_bytes))
        self.capacity = capacity_bytes

    def kmer_count(self, chunk_host, k, hist, window_size=0, lines_per_entry=4, header_char=ord("@"),
                   check_plus=True, trim_cr=-1, enc_mode=nv.ENC_ASCII_ACGT, lut_host=None, hist_mode=nv.HIST_AUTO):
        """chunk_host: CPU uint8 tensor (pinned for real overlap); hist: CUDA int64[n_bins]."""
        if chunk_host.is_cuda or chunk_host.dtype != torch.uint8:
            raise TypeError("chunk_host must be a CPU uint8 tensor")
        status = (ctypes.c_int64 * nv.ST_WORDS)()
        with torch.cuda.device(hist.device):
            check(lib().bnpk_pipeline_kmer_count_host_on(
                self._h, ctypes.c_void_p(chunk_host.data_ptr()), chunk_host.numel(), lines_per_entry, header_char,
                int(check_plus), trim_cr, enc_mode, ctypes.c_void_p(lut_host.data_ptr()) if lut_host is not None else None,
                k, window_size, hist.numel(), hist_mode, ptr(hist), ctypes.cast(status, ctypes.c_void_p), stream_ptr()))
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


def _format_fields(fields):
    """A host bnpk_field[3] of (name, sequence, quality); each a (base uint8, starts int64, lens int32, lut uint8[256]
    or None) of CUDA tensors, or None.  Returns (array, number of entries, device)."""
    arr = (nv.Field * 3)()
    n, dev = None, None
    for i, f in enumerate(fields):
        if f is None:
            continue
        base, starts, lens, lut = f
        base_p, base_bytes, starts_p, lens_p, rows = _rows_args(base, starts, lens)
        if lut is not None:
            _need_cuda(lut, "lut")
            if lut.dtype != torch.uint8 or lut.numel() != 256:
                raise TypeError("lut must be 256 uint8")
        if n is None:
            n, dev = rows, base.device
        if rows != n:
            raise ValueError("every field needs one row per entry")
        if any(t.device != dev for t in (base, starts, lens) + ((lut,) if lut is not None else ())):
            raise ValueError("the fields are on different devices")
        arr[i] = nv.Field(base_p.value, base_bytes, starts_p.value, lens_p.value, lut.data_ptr() if lut is not None else None)
    return arr, n or 0, dev


def format_offsets(fmt, line_width, fields, status=None):
    """int64[E+1] output offsets of the records (name, sequence, quality fields) in format ``fmt`` (nv.FMT_*) and the
    status tensor; with a sequence LUT, a sequence byte the LUT maps to 0 is reported in status[ST_BAD_BASE]."""
    arr, n, dev = _format_fields(fields)
    if dev is None:
        raise ValueError("format_offsets needs the name and sequence fields")
    with torch.cuda.device(dev):
        offsets = torch.empty(n + 1, dtype=torch.int64, device=dev)
        if status is None:
            status = nv.new_status(dev)
        ws = nv.workspace(max(n, 1), dev)
        check(lib().bnpk_format_offsets(fmt, line_width, n, ctypes.cast(arr, ctypes.c_void_p), ptr(offsets),
                                        ptr(status), ptr(ws), ws.numel(), stream_ptr()))
    return offsets, status


@_on_device
def format_records(fmt, line_width, fields, offsets, out_begin=0, out_end=None, out=None):
    """Bytes [out_begin, out_end) of the formatted records (default: all of them, offsets[-1] read back) into ``out``
    (uint8, at least out_end - out_begin bytes; allocated when None).  Returns ``out``."""
    _need_cuda(offsets, "offsets")
    arr, n, _ = _format_fields(fields)
    if out_end is None:
        out_end = int(offsets[-1].item())
    if out is None:
        out = torch.empty(max(out_end - out_begin, 0), dtype=torch.uint8, device=offsets.device)
    elif out.numel() < out_end - out_begin:
        raise ValueError("out is smaller than the range")
    check(lib().bnpk_format_records(fmt, line_width, n, ctypes.cast(arr, ctypes.c_void_p), ptr(offsets), out_begin,
                                    out_end, ptr(out) if out.numel() else None, stream_ptr()))
    return out


@_on_device
def delimited_columns(chunk, starts, lens, kinds, status=None):
    """The tab-separated columns of the lines (starts, lens) of ``chunk``, one nv.COL_* kind per column.  Returns
    (columns, status): per column None (COL_SKIP), (starts int64, lens int32) of text, int64 values or uint8 strand
    codes; the first fault is (line << 8 | column << 3 | nv.BAD_*) in status[ST_BAD_BASE]."""
    _rows_args(chunk, starts, lens)
    n, dev = lens.numel(), chunk.device
    if not 1 <= len(kinds) <= nv.MAX_COLUMNS:
        raise ValueError(f"1 to {nv.MAX_COLUMNS} columns")
    arr = (nv.Column * len(kinds))()
    cols = []
    for i, kind in enumerate(kinds):
        if kind == nv.COL_TEXT:
            col = (torch.empty(n, dtype=torch.int64, device=dev), torch.empty(n, dtype=torch.int32, device=dev))
            arr[i] = nv.Column(kind, col[0].data_ptr(), col[1].data_ptr())
        elif kind in (nv.COL_INT, nv.COL_INT_OR_DOT, nv.COL_STRAND):
            col = torch.empty(n, dtype=torch.uint8 if kind == nv.COL_STRAND else torch.int64, device=dev)
            arr[i] = nv.Column(kind, col.data_ptr(), None)
        else:
            col = None
            arr[i] = nv.Column(kind, None, None)
        cols.append(col)
    if status is None:
        status = nv.new_status(dev)
    check(lib().bnpk_delimited_columns(ptr(chunk), chunk.numel(), ptr(starts), ptr(lens), n,
                                       ctypes.cast(arr, ctypes.c_void_p), len(kinds), ptr(status), stream_ptr()))
    return cols, status


@_on_device
def name_lookup(base, starts, lens, names, name_offsets, status=None):
    """The index of each row's bytes in the sorted name table (names uint8, name_offsets int64[C+1]): int32, -1 for an
    unknown name, whose row is reported in status[ST_BAD_BASE].  Returns (ids, status)."""
    base_p, base_bytes, starts_p, lens_p, n = _rows_args(base, starts, lens)
    _need_cuda(names, "names")
    _need_cuda(name_offsets, "name_offsets")
    if names.dtype != torch.uint8 or name_offsets.dtype != torch.int64:
        raise TypeError("names must be uint8 and name_offsets int64")
    ids = torch.empty(n, dtype=torch.int32, device=base.device)
    if status is None:
        status = nv.new_status(base.device)
    check(lib().bnpk_name_lookup(base_p, base_bytes, starts_p, lens_p, n, ptr(names), ptr(name_offsets),
                                 name_offsets.numel() - 1, ptr(ids), ptr(status), stream_ptr()))
    return ids, status


def _interval_args(file, start, stop, ids, contigs):
    _need_cuda(file, "file")
    for t, name in ((start, "start"), (stop, "stop")):
        _need_cuda(t, name)
        if t.dtype != torch.int64:
            raise TypeError(f"{name} must be int64")
    if start.numel() != stop.numel() or (ids is not None and ids.numel() != start.numel()):
        raise ValueError("start, stop and ids differ in length")
    if ids is None:
        return [ptr(file), file.numel(), start.numel(), None, None, None, None, None, 0, ptr(start), ptr(stop)]
    offset, lenc, lenb, length = contigs
    for t, name, dt in ((ids, "ids", torch.int32), (offset, "contig_offset", torch.int64), (lenc, "lenc", torch.int32),
                        (lenb, "lenb", torch.int32), (length, "contig_len", torch.int64)):
        _need_cuda(t, name)
        if t.dtype != dt:
            raise TypeError(f"{name} must be {dt}")
    return [ptr(file), file.numel(), start.numel(), ptr(ids), ptr(offset), ptr(lenc), ptr(lenb), ptr(length),
            offset.numel(), ptr(start), ptr(stop)]


@_on_device
def interval_check(file, start, stop, ids=None, contigs=None, status=None):
    """The check pass of bnpk_interval_gather: (row_lens int32 = stop - start, 0 for a bad row; status with the first
    bad row in ST_BAD_BASE).  ``contigs`` = (offset int64, lenc int32, lenb int32, length int64) indexed by ``ids``
    (int32); without ids the file is one contig without line ends."""
    args = _interval_args(file, start, stop, ids, contigs)
    row_lens = torch.empty(start.numel(), dtype=torch.int32, device=file.device)
    if status is None:
        status = nv.new_status(file.device)
    check(lib().bnpk_interval_gather(*args, None, None, ptr(row_lens), None, None, ptr(status), stream_ptr()))
    return row_lens, status


@_on_device
def interval_copy(file, start, stop, offsets, total, ids=None, contigs=None, strand=None, complement_lut=None):
    """The copy pass: uint8[total], row r at offsets[r] (int64[R+1] of interval_check's row_lens), a row whose
    strand[r] (uint8) is not 0 reverse-complemented through ``complement_lut`` (uint8[256])."""
    args = _interval_args(file, start, stop, ids, contigs)
    _need_cuda(offsets, "offsets")
    if offsets.dtype != torch.int64 or offsets.numel() != start.numel() + 1:
        raise ValueError("offsets must be int64[R+1]")
    if strand is not None:
        _need_cuda(strand, "strand")
        _need_cuda(complement_lut, "complement_lut")
        if strand.dtype != torch.uint8 or strand.numel() != start.numel() or complement_lut.numel() != 256:
            raise ValueError("strand must be uint8[R] and complement_lut uint8[256]")
    out = torch.empty(total, dtype=torch.uint8, device=file.device)
    if total:
        check(lib().bnpk_interval_gather(*args, ptr(strand), ptr(complement_lut), None, ptr(offsets), ptr(out), None,
                                         stream_ptr()))
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


def _int64_args(*named):
    for t, name in named:
        _need_cuda(t, name)
        if t.dtype != torch.int64:
            raise TypeError(f"{name} must be int64")


@_on_device
def interval_events(start, stop, ids=None, contig_offset=None, contig_len=None, size=0, keys=True, glob=False,
                    status=None):
    """bnpk_interval_events: (keys int64[2R] or None, global start, global stop (or None), status).  ``ids`` (int32)
    index contig_offset / contig_len (int64; an offset < 0 leaves the contig out); without ids every row is on one
    contig of ``size``.  A bad row is reported in status[ST_BAD_BASE]."""
    _int64_args((start, "start"), (stop, "stop"))
    n = start.numel()
    if stop.numel() != n or (ids is not None and ids.numel() != n):
        raise ValueError("start, stop and ids differ in length")
    n_contigs = 0
    if ids is not None:
        _need_cuda(ids, "ids")
        _int64_args((contig_offset, "contig_offset"), (contig_len, "contig_len"))
        if ids.dtype != torch.int32 or contig_offset.numel() != contig_len.numel():
            raise TypeError("ids must be int32 and the contig columns of one length")
        n_contigs = contig_offset.numel()
    dev = start.device
    k = torch.empty(2 * n, dtype=torch.int64, device=dev) if keys else None
    gs, ge = (torch.empty(n, dtype=torch.int64, device=dev) for _ in range(2)) if glob else (None, None)
    if status is None:
        status = nv.new_status(dev)
    check(lib().bnpk_interval_events(ptr(start), ptr(stop), ptr(ids), ptr(contig_offset), ptr(contig_len), n_contigs,
                                     size, n, ptr(k), ptr(gs), ptr(ge), ptr(status), stream_ptr()))
    return k, gs, ge, status


@_on_device
def pileup_runs(sorted_keys, size, mode=nv.PILEUP_COUNT):
    """bnpk_pileup_runs on sorted event keys: (run_starts int64[K + 2], run_values int64[K + 1], n_runs int64[1]), the
    first n_runs + 1 starts and n_runs values valid (nothing is read back)."""
    _int64_args((sorted_keys, "keys"))
    n, dev = sorted_keys.numel(), sorted_keys.device
    starts = torch.empty(n + 2, dtype=torch.int64, device=dev)
    values = torch.empty(n + 1, dtype=torch.int64, device=dev)
    n_runs = torch.empty(1, dtype=torch.int64, device=dev)
    ws = nv.workspace(max(n, 1), dev)
    check(lib().bnpk_pileup_runs(ptr(sorted_keys), n, size, mode, ptr(starts), ptr(values), ptr(n_runs), ptr(ws),
                                 ws.numel(), stream_ptr()))
    return starts, values, n_runs


def _runs_args(run_starts, values):
    _int64_args((run_starts, "run_starts"), (values, "values"))
    if run_starts.numel() != values.numel() + 1 or values.numel() < 1:
        raise ValueError("a track is R >= 1 values and R + 1 run starts")
    return ptr(run_starts), ptr(values), values.numel()


@_on_device
def runs_reduce(run_starts, values, q_start, q_stop, mode):
    """bnpk_runs_reduce: int64[Q], one reduction (nv.RUNS_*) per query [q_start, q_stop); no synchronisation."""
    runs = _runs_args(run_starts, values)
    _int64_args((q_start, "q_start"), (q_stop, "q_stop"))
    if q_start.numel() != q_stop.numel():
        raise ValueError("q_start and q_stop differ in length")
    n, dev = q_start.numel(), q_start.device
    out = torch.empty(n, dtype=torch.int64, device=dev)
    scratch = torch.empty(3 * n + 1, dtype=torch.int64, device=dev)
    ws = nv.workspace(max(n, 1), dev)
    check(lib().bnpk_runs_reduce(*runs, ptr(q_start), ptr(q_stop), n, mode, ptr(out), ptr(scratch), ptr(ws),
                                 ws.numel(), stream_ptr()))
    return out


@_on_device
def runs_extract(run_starts, values, q_start, out_offsets, total):
    """bnpk_runs_extract: int64[total], query q's values at out_offsets[q] (int64[Q + 1])."""
    runs = _runs_args(run_starts, values)
    _int64_args((q_start, "q_start"), (out_offsets, "out_offsets"))
    if out_offsets.numel() != q_start.numel() + 1:
        raise ValueError("out_offsets must be int64[Q + 1]")
    out = torch.empty(total, dtype=torch.int64, device=q_start.device)
    if total:
        check(lib().bnpk_runs_extract(*runs, ptr(q_start), q_start.numel(), ptr(out_offsets), ptr(out), stream_ptr()))
    return out


@_on_device
def interval_merge(start, stop, same_prev=None, distance=0, status=None):
    """bnpk_interval_merge: (out_rows int64[R], out_stops int64[R], n_out int64[1], status), the first n_out entries
    valid; a start that decreases inside a segment is reported in status[ST_BAD_BASE]."""
    _int64_args((start, "start"), (stop, "stop"))
    n, dev = start.numel(), start.device
    if stop.numel() != n or (same_prev is not None and (same_prev.numel() != n or same_prev.dtype != torch.uint8)):
        raise ValueError("start, stop and same_prev (uint8) differ in length")
    if same_prev is not None:
        _need_cuda(same_prev, "same_prev")
    rows, stops = (torch.empty(n, dtype=torch.int64, device=dev) for _ in range(2))
    n_out = torch.empty(1, dtype=torch.int64, device=dev)
    if status is None:
        status = nv.new_status(dev)
    ws = nv.workspace(max(n, 1), dev)
    check(lib().bnpk_interval_merge(ptr(start), ptr(stop), ptr(same_prev), n, max(int(distance), 0), ptr(rows),
                                    ptr(stops), ptr(n_out), ptr(status), ptr(ws), ws.numel(), stream_ptr()))
    return rows, stops, n_out, status


@_on_device
def rows_equal_prev(base, starts, lens):
    """bnpk_rows_equal_prev: uint8[R], 1 where a row's bytes equal the previous row's."""
    args = _rows_args(base, starts, lens)
    flag = torch.empty(lens.numel(), dtype=torch.uint8, device=base.device)
    check(lib().bnpk_rows_equal_prev(*args, ptr(flag), stream_ptr()))
    return flag


@_on_device
def runs_combine(a_starts, a_values, b_starts, b_values, op):
    """bnpk_runs_combine: (run_starts int64[Ra + Rb + 1], run_values int64[Ra + Rb], n_runs int64[1]), the canonical
    runs of op(A, B) (nv.OP_*) of two tracks of one size, the first n_runs + 1 starts and n_runs values valid (nothing
    is read back)."""
    _int64_args((a_starts, "a_starts"), (a_values, "a_values"), (b_starts, "b_starts"), (b_values, "b_values"))
    if a_starts.numel() != a_values.numel() + 1 or b_starts.numel() != b_values.numel() + 1:
        raise ValueError("a track is R values and R + 1 run starts")
    n, dev = a_values.numel() + b_values.numel(), a_starts.device
    starts = torch.empty(n + 1, dtype=torch.int64, device=dev)
    values = torch.empty(max(n, 1), dtype=torch.int64, device=dev)
    n_runs = torch.empty(1, dtype=torch.int64, device=dev)
    ws = nv.workspace(max(n, 1), dev)
    check(lib().bnpk_runs_combine(ptr(a_starts), ptr(a_values), a_values.numel(), ptr(b_starts), ptr(b_values),
                                  b_values.numel(), op, ptr(starts), ptr(values), ptr(n_runs), ptr(ws), ws.numel(),
                                  stream_ptr()))
    return starts, values, n_runs


@_on_device
def interval_intersect(start, stop, same_prev=None, rows=True):
    """bnpk_interval_intersect over rows sorted by start and, separately, their stops sorted (inside each segment of
    ``same_prev``, uint8): (out_rows int64[R] or None, out_stops int64[R] or None, n_out int64[1], overlap int64[1]),
    the first n_out rows valid.  ``rows=False`` counts the pairs and sums their overlaps only."""
    _int64_args((start, "start"), (stop, "stop"))
    n, dev = start.numel(), start.device
    if stop.numel() != n or (same_prev is not None and (same_prev.numel() != n or same_prev.dtype != torch.uint8)):
        raise ValueError("start, stop and same_prev (uint8) differ in length")
    if same_prev is not None:
        _need_cuda(same_prev, "same_prev")
    out_rows, out_stops = (torch.empty(n, dtype=torch.int64, device=dev) for _ in range(2)) if rows else (None, None)
    n_out, overlap = (torch.empty(1, dtype=torch.int64, device=dev) for _ in range(2))
    ws = nv.workspace(max(n, 1), dev)
    check(lib().bnpk_interval_intersect(ptr(start), ptr(stop), ptr(same_prev), n, ptr(out_rows), ptr(out_stops),
                                        ptr(n_out), ptr(overlap), ptr(ws), ws.numel(), stream_ptr()))
    return out_rows, out_stops, n_out, overlap


@_on_device
def runs_to_intervals(run_starts, values, contig_ends, mode=nv.RUNS_TO_NONZERO):
    """bnpk_runs_to_intervals: the rows of a global track cut at the contig ends (int64[C + 1], strictly increasing
    from 0 to the size): (contig int32, start int64, stop int64, value int64 or None, n_out int64[1]), each of capacity
    R + C, the first n_out rows valid (nothing is read back).  nv.RUNS_TO_NONZERO: the stretches of non-zero value;
    nv.RUNS_TO_ALL: every run, with its value."""
    _int64_args((run_starts, "run_starts"), (values, "values"), (contig_ends, "contig_ends"))
    if run_starts.numel() != values.numel() + 1:
        raise ValueError("a track is R values and R + 1 run starts")
    if contig_ends.numel() < 2:
        raise ValueError("contig_ends holds 0 and the end of every contig")
    n, c, dev = values.numel(), contig_ends.numel() - 1, run_starts.device
    contig = torch.empty(n + c, dtype=torch.int32, device=dev)
    start, stop = (torch.empty(n + c, dtype=torch.int64, device=dev) for _ in range(2))
    value = torch.empty(n + c, dtype=torch.int64, device=dev) if mode == nv.RUNS_TO_ALL else None
    n_out = torch.empty(1, dtype=torch.int64, device=dev)
    ws = nv.workspace(max(n, 1), dev)
    check(lib().bnpk_runs_to_intervals(ptr(run_starts), ptr(values), n, ptr(contig_ends), c, mode, ptr(contig),
                                       ptr(start), ptr(stop), ptr(value), ptr(n_out), ptr(ws), ws.numel(),
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
            base_p, base_bytes, starts_p, lens_p, n = _rows_args(*data)
            arr[i] = nv.OutColumn(kind, base_p.value, base_bytes, starts_p.value, lens_p.value)
            d = data[0].device
        elif kind in (nv.COL_INT, nv.COL_STRAND):
            _need_cuda(data, "column")
            want = torch.int64 if kind == nv.COL_INT else torch.uint8
            if data.dtype != want:
                raise TypeError(f"an {'INT' if kind == nv.COL_INT else 'STRAND'} column must be {want}")
            arr[i] = nv.OutColumn(kind, data.data_ptr() or None, 0, None, None)
            n, d = data.numel(), data.device
        else:
            raise ValueError(f"unknown column kind {kind}")
        if rows is None:
            rows, dev = n, d
        if n != rows:
            raise ValueError(f"the columns differ in length ({rows} and {n} rows)")
        if d != dev:
            raise ValueError("the columns are on different devices")
    return arr, rows, dev


def delimited_offsets(columns, status=None):
    """bnpk_delimited_offsets: (int64[E + 1] line offsets, status); a strand code above 2 is reported in
    status[ST_BAD_BASE] as (line << 8 | column << 3 | nv.BAD_STRAND)."""
    arr, n, dev = _out_columns(columns)
    with torch.cuda.device(dev):
        offsets = torch.empty(n + 1, dtype=torch.int64, device=dev)
        if status is None:
            status = nv.new_status(dev)
        ws = nv.workspace(max(n, 1), dev)
        check(lib().bnpk_delimited_offsets(ctypes.cast(arr, ctypes.c_void_p), len(columns), n, ptr(offsets),
                                           ptr(status), ptr(ws), ws.numel(), stream_ptr()))
    return offsets, status


@_on_device
def delimited_format(columns, offsets, out_begin=0, out_end=None, out=None):
    """Bytes [out_begin, out_end) of the lines (default: all, offsets[-1] read back) into ``out`` (uint8, at least
    out_end - out_begin bytes; allocated when None).  Returns ``out``."""
    _need_cuda(offsets, "offsets")
    arr, n, _ = _out_columns(columns)
    if offsets.dtype != torch.int64 or offsets.numel() != n + 1:
        raise ValueError("offsets must be int64[E + 1]")
    if out_end is None:
        out_end = int(offsets[-1].item())
    if out is None:
        out = torch.empty(max(out_end - out_begin, 0), dtype=torch.uint8, device=offsets.device)
    elif out.numel() < out_end - out_begin:
        raise ValueError("out is smaller than the range")
    check(lib().bnpk_delimited_format(ctypes.cast(arr, ctypes.c_void_p), len(columns), n, ptr(offsets), out_begin,
                                      out_end, ptr(out) if out.numel() else None, stream_ptr()))
    return out
