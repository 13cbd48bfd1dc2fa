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
from ..datatypes import Bed6, BedGraph, GFFEntry, GTFEntry, Interval, NarrowPeak, StrandedInterval
from ..encoded_array import EncodedArray, EncodedRaggedArray, BaseEncoding
from ..encodings import StrandEncoding
from .buffers import FieldView, _to_device_bytes
from .exceptions import FormatException, IncompleteEntryException

_FAULTS = {nv.BAD_TABS: "Irregular number of delimiters per line",
           nv.BAD_COLUMNS: "Too few columns for the record type",
           nv.BAD_INT: "Invalid integer (an optional sign and 1 to 18 digits)",
           nv.BAD_STRAND: "Invalid strand (one of '+', '-', '.')",
           nv.BAD_FLOAT: "Invalid number ([+-]? (digits ['.' digits?] | '.' digits) ([eE] [+-]? digits)?, at most 19 "
                         "significant digits; nan and inf are not read)"}


class DelimitedBuffer:
    DELIMITER = "\t"
    COMMENT = "#"
    n_lines_per_entry = 1
    dataclass = None
    _kinds = ()                 # nv.COL_* of the record type's fields, in column order
    _float_columns = ()         # the COL_TEXT columns read as float64 values (bnpk_parse_float)

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
        floats = {c: cls._parse_floats(chunk, cols[c], c, status) for c in cls._float_columns}
        # the one synchronisation of the columns: the first fault and the chunk's size
        st, last_end = ops.read_back(status, starts[-1:] + lens[-1:])
        if st.fault is not None:
            line, col, kind = st.column_fault()
            raise FormatException(f"{_FAULTS.get(kind, 'Invalid line')} (column {col})", line_number=line)
        data = chunk[:last_end + 1]
        fields = []
        for i, (kind, col) in enumerate(zip(cls._kinds, cols)):
            if i in floats:
                fields.append(floats[i])
            elif kind == nv.COL_TEXT:
                fields.append(FieldView(data, col[1], col[0]))
            elif kind == nv.COL_STRAND:
                fields.append(EncodedArray(col, StrandEncoding))
            else:
                fields.append(col)
        return cls(data, n_lines, fields)

    @staticmethod
    def _parse_floats(chunk, view, column, status):
        """The float64 values of one text column (bnpk_parse_float into the chunk's status block, no synchronisation).
        A line without the column leaves its view unwritten: the parse is kept inside the chunk, and the column fault
        of such a line is smaller than any value fault of it."""
        from .decimal import pow5_table
        v_start = view[0].clamp(0, chunk.numel())
        v_lens = torch.minimum(view[1].clamp(min=0).to(torch.int64), chunk.numel() - v_start).to(torch.int32)
        values, _ = ops.parse_float(chunk, v_start, v_lens, column, pow5_table(chunk.device), status)
        return values

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
    """bedGraph for writing: chromosome, start, stop and an integer value (a float value cannot be written yet).  It
    does not read: BedGraphBuffer reads bedGraph, with float64 values."""
    dataclass = BedGraph

    @classmethod
    def from_raw_buffer(cls, chunk, header_data=None):
        raise NotImplementedError("BdgBuffer writes bedGraph; read it with BedGraphBuffer")


class BedGraphBuffer(BdgBuffer):
    """bedGraph read on the device (delimited_buffers.py BedGraphBuffer): chromosome, start, stop and a float64 value.
    The columns are read as a BED chunk's are, then the value column's text is parsed by bnpk_parse_float into the same
    status block, so a chunk takes the two synchronisations of a BED chunk.  Each value equals Python's float(text);
    the grammar is [+-]? (digits ['.' digits?] | '.' digits) ([eE] [+-]? digits)? of at most 19 significant digits,
    so nan, inf and longer significands raise FormatException naming the line.  Leading ``#``, ``track`` and
    ``browser`` lines are the header."""
    _kinds = (nv.COL_TEXT, nv.COL_INT, nv.COL_INT, nv.COL_TEXT)
    _float_columns = (3,)

    from_raw_buffer = DelimitedBuffer.__dict__["from_raw_buffer"]       # read as every delimited buffer; BdgBuffer's refuses

    @classmethod
    def read_header(cls, file_object):
        header = []
        for line in file_object:
            if not (line.startswith(b"#") or line.startswith(b"track") or line.startswith(b"browser")):
                file_object.seek(-len(line), 1)
                break
            header.append(line.decode("utf-8"))
        return "".join(header)


class NarrowPeakBuffer(DelimitedBuffer):
    """MACS2 narrowPeak read on the device (delimited_buffers.py NarrowPeakBuffer): the six BED6 columns, signal_value,
    p_value and q_value (float64) and summit (int64).  The columns are read as a BED chunk's are, then the three float
    columns' text is parsed by bnpk_parse_float into the same status block, so a chunk takes the two synchronisations
    of a BED chunk; a bad value raises FormatException naming its line (the grammar of BedGraphBuffer).  Read only."""
    dataclass = NarrowPeak
    _kinds = (nv.COL_TEXT, nv.COL_INT, nv.COL_INT, nv.COL_TEXT, nv.COL_INT_OR_DOT, nv.COL_STRAND, nv.COL_TEXT,
              nv.COL_TEXT, nv.COL_TEXT, nv.COL_INT)
    _float_columns = (6, 7, 8)

    @classmethod
    def formatted(cls, entries):
        raise NotImplementedError("writing narrowPeak is not supported: it is read only")

    from_data = formatted


_GTF_KINDS = (nv.COL_TEXT, nv.COL_TEXT, nv.COL_TEXT, nv.COL_INT, nv.COL_INT, nv.COL_TEXT, nv.COL_STRAND, nv.COL_TEXT,
              nv.COL_TEXT)


class GTFBuffer(DelimitedBuffer):
    """delimited_buffers.py GTFBuffer: the nine GTF columns (GTFEntry).  Read only."""
    dataclass = GTFEntry
    _kinds = _GTF_KINDS

    @classmethod
    def formatted(cls, entries):
        raise NotImplementedError(f"writing {cls.__name__[:3]} is not supported")

    from_data = formatted


class GFFBuffer(GTFBuffer):
    """delimited_buffers.py GFFBuffer (DelimitedBufferWithInernalComments): the GTF columns with GFF3 attributes, and
    comment lines inside the chunk (``##sequence-region`` lines, ``###`` separators) dropped after the line split.
    Two synchronisations: the comment count, then the columns.  A FormatException counts the chunk's lines, comments
    included."""
    dataclass = GFFEntry

    @classmethod
    def from_raw_buffer(cls, chunk, header_data=None):
        chunk = _to_device_bytes(chunk)
        n_lines = ops.count_byte(chunk, 10) if chunk.numel() else 0
        if n_lines == 0:
            raise IncompleteEntryException("No complete line in the buffer. Try increasing chunk_size.")
        starts, lens, _ = ops.line_split(chunk, 1, 0, 0, ord(cls.COMMENT), False, 0, max_rows=n_lines)
        keep = ((chunk[starts] != ord(cls.COMMENT)) | (lens == 0)).to(torch.uint8)
        n_keep, last_end = ops.read_back(keep.sum(), starts[-1:] + lens[-1:])
        data = chunk[:last_end + 1]
        lines = torch.nonzero_static(keep, size=n_keep).reshape(-1)
        if n_keep == 0:
            empty = torch.zeros(0, dtype=torch.int64, device=chunk.device)
            buf = cls(data, 0, [FieldView(data, lens[:0], starts[:0]) if k == nv.COL_TEXT else
                                EncodedArray(empty.to(torch.uint8), StrandEncoding) if k == nv.COL_STRAND else empty
                                for k in cls._kinds])
            buf._n_chunk_lines = n_lines
            return buf
        cols, status = ops.delimited_columns(chunk, starts[lines], lens[lines], cls._kinds)
        st, = ops.read_back(status)
        if st.fault is not None:
            line, col, kind = st.column_fault()
            raise FormatException(f"{_FAULTS.get(kind, 'Invalid line')} (column {col})",
                                  line_number=int(lines[line].item()))
        fields = []
        for kind, col in zip(cls._kinds, cols):
            if kind == nv.COL_TEXT:
                fields.append(FieldView(data, col[1], col[0]))
            elif kind == nv.COL_STRAND:
                fields.append(EncodedArray(col, StrandEncoding))
            else:
                fields.append(col)
        buf = cls(data, n_keep, fields)
        buf._n_chunk_lines = n_lines
        return buf

    @property
    def n_lines(self) -> int:
        """The chunk's lines, comments included (the reader counts a FormatException's line number with them)."""
        return getattr(self, "_n_chunk_lines", self._n_lines)


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
        self.size, st = ops.read_back(self.offsets[-1:], status)
        if st.fault is not None:
            line, col, _ = st.column_fault()
            raise ValueError(f"line {line}: the {entries._fields[col]} column holds a strand code that is not "
                             "'+', '-' or '.'")

    def slice(self, begin, end, out=None):
        return ops.delimited_format(self.columns, self.offsets, begin, end, out)
