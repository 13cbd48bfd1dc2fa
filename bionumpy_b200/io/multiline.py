"""Multi-line FASTA on the device (mirror of bionumpy/io/multiline_buffer.py:15-109).

  from_raw_buffer : every newline-terminated line of the chunk via K1 (lines_per_entry = 1), header lines are
                    the ones that start with '>', the buffer is cut at the start of the last header line
                    (multiline_buffer.py:89-101)
  get_data        : headers are (chunk, starts, lens) views; the sequence lines of each entry are joined by the
                    row-driven copy kernel (K2 with an identity LUT) -- the reference's boolean-mask gather
                    (multiline_buffer.py:46-62) -- giving one contiguous row per entry.
The per-line bookkeeping (which line is a header, which entry a line belongs to, entry lengths, the compacted list of
sequence lines) is two small kernels and a device scan (bnpk_multiline_flags, bnpk_row_offsets, bnpk_multiline_entries)."""
import torch

from .. import _native as nv
from .. import ops
from ..datatypes import SequenceEntry
from ..encoded_array import EncodedArray, EncodedRaggedArray, BaseEncoding
from .buffers import FieldView, _to_device_bytes
from .exceptions import IncompleteEntryException

_identity_luts = {}


def _identity_lut(device):
    key = (device.type, device.index)
    if key not in _identity_luts:
        _identity_luts[key] = torch.arange(256, dtype=torch.uint8, device=device)
    return _identity_luts[key]


class CudaMultiLineFastaBuffer:
    _new_entry_marker = ">"
    n_characters_per_line = 80
    dataclass = SequenceEntry
    SKIP_LAZY = True

    def __init__(self, data, line_starts, line_lens, is_header, trim_cr=False):
        self._data = data                    # device bytes, complete entries only
        self._line_starts, self._line_lens, self._is_header = line_starts, line_lens, is_header
        self._trim_cr = trim_cr
        # entry index of every line = headers before it (device scan, K-row_offsets); the total is the entry count
        self._hdr_before = ops.row_offsets(is_header.contiguous(), 0)
        self._n_entries = int(self._hdr_before[-1].item())
        self._cache = None

    # ---- protocol ---------------------------------------------------------------------------------
    @classmethod
    def read_header(cls, file_object):
        return None

    @classmethod
    def modify_class_with_header_data(cls, header_data):
        return cls

    @classmethod
    def _lines(cls, chunk):
        """(starts, lens) of every newline-terminated line of chunk[:-1] (multiline_buffer.py:92)."""
        body = chunk[:-1] if chunk.numel() else chunk
        n_lines = ops.count_byte(body, 10) if body.numel() else 0
        starts, lens, _ = ops.line_split(body, 1, 0, 0, ord(">"), False, 0, max_rows=n_lines)
        return starts, lens

    @classmethod
    def contains_complete_entry(cls, chunks):
        assert len(chunks) == 1
        try:
            return True, cls.from_raw_buffer(chunks[0])
        except IncompleteEntryException:
            return False

    @classmethod
    def from_raw_buffer(cls, chunk, header_data=None):
        assert header_data is None, header_data
        chunk = _to_device_bytes(chunk)
        assert chunk.numel() and int(chunk[0].item()) == ord(">"), "multi-line FASTA chunk must start with '>'"
        starts, lens = cls._lines(chunk)
        # header flags, the last newline that is followed by an entry start (multiline_buffer.py:93), '\r' probe: one kernel
        is_header, out2 = ops.multiline_flags(chunk, starts, lens)
        keep, has_cr = (int(x) for x in out2.cpu().tolist())          # the one synchronisation of this buffer
        if keep == 0:
            raise IncompleteEntryException("No complete entry found in multi-line FASTA buffer")
        size = int((starts[keep - 1] + lens[keep - 1]).item()) + 1      # start of the last (incomplete) entry
        return cls(chunk[:size], starts[:keep], lens[:keep], is_header[:keep], bool(has_cr))

    @property
    def size(self) -> int:
        return self._data.numel()

    @property
    def n_lines(self) -> int:
        # the reference keeps new_lines[:new_entries[-1]] (multiline_buffer.py:99-101): the newline that precedes the
        # next entry's header is not counted
        return max(self._line_starts.numel() - 1, 0)

    @property
    def data(self):
        return EncodedArray(self._data, BaseEncoding)

    def count_entries(self) -> int:
        return self._n_entries

    def __len__(self):
        return self._n_entries

    def _materialise(self):
        if self._cache is None:
            h_starts, h_lens, s_starts, s_lens, entry_lens = ops.multiline_entries(
                self._data, self._line_starts, self._line_lens, self._is_header, self._hdr_before, self._n_entries,
                self._trim_cr)
            flat, _, _ = ops.rows_encode(self._data, s_starts, s_lens, nv.ENC_LUT, _identity_lut(self._data.device))
            names = FieldView(self._data, h_lens, h_starts)
            seqs = EncodedRaggedArray(EncodedArray(flat, BaseEncoding), entry_lens.to(torch.int32))
            self._cache = (names, seqs)
        return self._cache

    def get_field_by_number(self, i, t=None):
        return self._materialise()[i]

    def get_data(self):
        return self.dataclass.lazy(self)

    # ---- writing (MultiLineFastaBuffer.from_data, io/multiline_buffer.py:67-86) --------------------------------------
    @classmethod
    def _write_format(cls):
        return nv.FMT_FASTA_WRAPPED, int(cls.n_characters_per_line)

    @classmethod
    def formatted(cls, entries):
        from .write import formatted_entries
        return formatted_entries(entries, *cls._write_format())

    @classmethod
    def from_data(cls, entries):
        """The records as FASTA with n_characters_per_line bases per line: a device EncodedArray.  An entry with an
        empty sequence is its header line alone."""
        from .write import format_entries
        return format_entries(entries, *cls._write_format())

    @classmethod
    def join_fields(cls, fields):
        from .write import join_fields
        return join_fields(fields, *cls._write_format())


MultiLineFastaBuffer = CudaMultiLineFastaBuffer
