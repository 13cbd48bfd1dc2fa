"""BED on the device (mirror of bionumpy/io/delimited_buffers.py:29-316 for BedBuffer and Bed6Buffer).

  from_raw_buffer : every newline-terminated line of the chunk via K1 (lines_per_entry = 1), then the columns the
                    record type names via bnpk_delimited_columns: text columns as (chunk, starts, lens) views, integers
                    as int64, strand as StrandEncoding codes.  The chunk is cut after its last newline; the first fault
                    of the chunk is raised as the reference's FormatException(line_number).
  get_data        : the record type, built lazily from those columns."""
import torch

from .. import _native as nv
from .. import ops
from ..datatypes import Bed6, Interval
from ..encoded_array import EncodedArray, BaseEncoding
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
    def from_data(cls, entries):
        raise NotImplementedError("writing BED is not supported")


class BedBuffer(DelimitedBuffer):
    """delimited_buffers.py BedBuffer: chromosome, start, stop."""
    dataclass = Interval
    _kinds = (nv.COL_TEXT, nv.COL_INT, nv.COL_INT)


class Bed6Buffer(DelimitedBuffer):
    """delimited_buffers.py Bed6Buffer: chromosome, start, stop, name, score (. = 0), strand."""
    dataclass = Bed6
    _kinds = (nv.COL_TEXT, nv.COL_INT, nv.COL_INT, nv.COL_TEXT, nv.COL_INT_OR_DOT, nv.COL_STRAND)
