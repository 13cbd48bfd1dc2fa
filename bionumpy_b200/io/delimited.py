"""BED on the device (mirror of bionumpy/io/delimited_buffers.py:29-316 for BedBuffer and Bed6Buffer).

  from_raw_buffer : every newline-terminated line of the chunk via K1 (lines_per_entry = 1), then the columns the
                    record type names via bnpk_delimited_columns: text columns as (chunk, starts, lens) views, integers
                    as int64, strand as StrandEncoding codes.  The chunk is cut after its last newline; the first fault
                    of the chunk is raised as the reference's FormatException(line_number).
  get_data        : the record type, built lazily from those columns.
  from_data       : the record's own fields as tab-separated lines, formatted on the device (bnpk_delimited_offsets /
                    bnpk_delimited_format): text as it is, integers in decimal, strand as '+', '-' or '.'."""
import torch

from .. import _native as nv
from .. import ops
from ..datatypes import Bed6, BedGraph, Interval, StrandedInterval
from ..encoded_array import EncodedArray, EncodedRaggedArray, BaseEncoding
from ..encodings import StrandEncoding
from .buffers import FieldView, _to_device_bytes
from .exceptions import FormatException, IncompleteEntryException

_FAULTS = {nv.BAD_TABS: "Irregular number of delimiters per line",
           nv.BAD_COLUMNS: "Too few columns for the record type",
           nv.BAD_INT: "Invalid integer (an optional sign and 1 to 18 digits)",
           nv.BAD_STRAND: "Invalid strand (one of '+', '-', '.')"}


class DelimitedBuffer:
    DELIMITER = "\t"
    COMMENT = "#"
    n_lines_per_entry = 1
    dataclass = None
    _kinds = ()                 # nv.COL_* of the record type's fields, in column order

    def __init__(self, data, n_lines, fields):
        self._data = data       # device bytes, complete lines only
        self._n_lines = n_lines
        self._fields = fields

    # ---- protocol ---------------------------------------------------------------------------------
    @classmethod
    def read_header(cls, file_object):
        """file_buffers.py:135-165: the leading comment lines; the file is left at the first other line."""
        header = []
        comment = ord(cls.COMMENT)
        for line in file_object:
            if line[0] != comment:
                file_object.seek(-len(line), 1)
                break
            header.append(line.decode("utf-8"))
        return "".join(header)

    @classmethod
    def modify_class_with_header_data(cls, header_data):
        return cls

    @classmethod
    def contains_complete_entry(cls, chunks):
        assert len(chunks) == 1
        try:
            return True, cls.from_raw_buffer(chunks[0])
        except IncompleteEntryException:
            return False

    @classmethod
    def from_raw_buffer(cls, chunk, header_data=None):
        chunk = _to_device_bytes(chunk)
        n_lines = ops.count_byte(chunk, 10) if chunk.numel() else 0
        if n_lines == 0:
            raise IncompleteEntryException("No complete line in the buffer. Try increasing chunk_size.")
        starts, lens, _ = ops.line_split(chunk, 1, 0, 0, ord(cls.COMMENT), False, 0, max_rows=n_lines)
        cols, status = ops.delimited_columns(chunk, starts, lens, cls._kinds)
        # the one synchronisation of the columns: the first fault and the chunk's size
        fault, last_end = (int(x) for x in torch.cat([status[nv.ST_BAD_BASE:nv.ST_BAD_BASE + 1],
                                                      starts[-1:] + lens[-1:]]).cpu().tolist())
        if fault != nv.INT64_MAX:
            line, col, kind = fault >> 8, (fault >> 3) & 31, fault & 7
            raise FormatException(f"{_FAULTS.get(kind, 'Invalid line')} (column {col})", line_number=line)
        data = chunk[:last_end + 1]
        fields = []
        for kind, col in zip(cls._kinds, cols):
            if kind == nv.COL_TEXT:
                fields.append(FieldView(data, col[1], col[0]))
            elif kind == nv.COL_STRAND:
                fields.append(EncodedArray(col, StrandEncoding))
            else:
                fields.append(col)
        return cls(data, n_lines, fields)

    @property
    def size(self) -> int:
        return self._data.numel()

    @property
    def n_lines(self) -> int:
        return self._n_lines

    @property
    def data(self):
        return EncodedArray(self._data, BaseEncoding)

    def count_entries(self) -> int:
        return self._n_lines

    def __len__(self):
        return self._n_lines

    def get_field_by_number(self, i, t=None):
        return self._fields[i]

    def get_data(self):
        return self.dataclass.lazy(self)

    @classmethod
    def formatted(cls, entries):
        """The text of a record chunk, its size known and any byte range formatted on demand (the writer's protocol)."""
        return DelimitedText(entries)

    @classmethod
    def from_data(cls, entries):
        """The records as tab-separated lines of their own fields (delimited_buffers.py:150-160): a device
        EncodedArray.  Bed6 records give six columns whatever the buffer type."""
        text = DelimitedText(entries)
        return EncodedArray(text.slice(0, text.size), BaseEncoding)


class BedBuffer(DelimitedBuffer):
    """delimited_buffers.py BedBuffer: chromosome, start, stop."""
    dataclass = Interval
    _kinds = (nv.COL_TEXT, nv.COL_INT, nv.COL_INT)


class Bed6Buffer(DelimitedBuffer):
    """delimited_buffers.py Bed6Buffer: chromosome, start, stop, name, score (. = 0), strand."""
    dataclass = Bed6
    _kinds = (nv.COL_TEXT, nv.COL_INT, nv.COL_INT, nv.COL_TEXT, nv.COL_INT_OR_DOT, nv.COL_STRAND)


class BdgBuffer(DelimitedBuffer):
    """bedGraph: chromosome, start, stop and an integer value.  Written only: the reference reads bedGraph values as
    floats, and this package has no float tracks."""
    dataclass = BedGraph

    @classmethod
    def from_raw_buffer(cls, chunk, header_data=None):
        raise NotImplementedError("reading bedGraph is not supported: its values are floats")


_WRITTEN = (Interval, StrandedInterval, Bed6, BedGraph)


def _column(entries, field):
    """(nv.COL_*, tensors) of one field of a record chunk."""
    from .write import _view
    value = getattr(entries, field)
    if isinstance(value, EncodedRaggedArray):
        if not value.encoding.is_base_encoding():
            raise TypeError(f"the {field} column must be text, got {value.encoding}")
        return nv.COL_TEXT, _view(value)
    if isinstance(value, EncodedArray):
        if value.encoding != StrandEncoding:
            raise TypeError(f"the {field} column must be text or strand codes, got {value.encoding}")
        return nv.COL_STRAND, value.raw().reshape(-1).to(torch.uint8).contiguous()
    if not isinstance(value, torch.Tensor):
        raise TypeError(f"the {field} column must be a tensor, got {type(value).__name__}")
    if value.is_floating_point() or value.is_complex():
        raise TypeError(f"the {field} column holds {value.dtype}: only integer values are written")
    if not value.is_cuda:
        raise nv.NativeLibraryError("writing needs CUDA tensors: bionumpy_b200 has no CPU fallback")
    return nv.COL_INT, value.reshape(-1).to(torch.int64).contiguous()


class DelimitedText:
    """The tab-separated text of a record chunk: line offsets on the device and the size, read with the first bad
    strand code in one synchronisation; ``slice(a, b, out)`` formats bytes [a, b)."""

    def __init__(self, entries):
        if not isinstance(entries, _WRITTEN):
            raise TypeError(f"cannot write {type(entries).__name__} as delimited text: "
                            f"{', '.join(t.__name__ for t in _WRITTEN)} are written")
        self.columns = [_column(entries, f) for f in entries._fields]
        self.offsets, status = ops.delimited_offsets(self.columns)
        self.size, fault = (int(x) for x in torch.cat([self.offsets[-1:],
                                                       status[nv.ST_BAD_BASE:nv.ST_BAD_BASE + 1]]).cpu().tolist())
        if fault != nv.INT64_MAX:
            line, col = fault >> 8, (fault >> 3) & 31
            raise ValueError(f"line {line}: the {entries._fields[col]} column holds a strand code that is not "
                             "'+', '-' or '.'")

    def slice(self, begin, end, out=None):
        return ops.delimited_format(self.columns, self.offsets, begin, end, out)
