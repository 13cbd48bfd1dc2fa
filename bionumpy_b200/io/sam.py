"""SAM on the device (mirror of bionumpy/io/buffers/sam.py SAMBuffer).

  from_raw_buffer : every newline-terminated line of the chunk via K1 (lines_per_entry = 1), then the 11 mandatory
                    columns and the extra text of every line via K16 bnpk_sam_columns, read back with the chunk's size
                    in one synchronisation (after the line census, as BedBuffer).  The chunk is cut after its last
                    newline; the first fault of the chunk raises FormatException(line_number).
  get_data        : SAMEntry, text columns as (chunk, starts, lens) views and integers as int64 rows of the field
                    matrix, no copy.

The header is the leading '@' lines (read_header, as DelimitedBuffer with COMMENT = '@').  The CIGAR is text here and
is not validated when a SAMEntry is read; bnp.alignments.parse_cigar, alignment_to_interval and SAMIntervalBuffer
parse it (bnpk_cigar_count / bnpk_cigar_unpack).

Deviations from the reference: a line with fewer than 11 columns, or a FLAG, POS, MAPQ, PNEXT or TLEN that is not an
optional sign and 1 to 18 digits, raises FormatException (the reference misaligns or crashes); SAMIntervalBuffer leaves
out records whose RNAME is '*', as BamIntervalBuffer leaves out refID -1."""
import torch

from .. import _native as nv
from .. import ops
from ..datatypes import Bed6, SAMEntry
from ..encoded_array import EncodedArray
from ..encodings import StrandEncoding
from .buffers import FieldView, _to_device_bytes
from .delimited import DelimitedBuffer
from .exceptions import FormatException, IncompleteEntryException

_FAULTS = {nv.BAD_COLUMNS: "Too few columns for a SAM line (11 are mandatory)",
           nv.BAD_INT: "Invalid integer (an optional sign and 1 to 18 digits)",
           nv.BAD_CIGAR: "Invalid CIGAR ('*', or ops of 1 to 9 digits and one of MIDNSHP=X)"}

# SAMEntry field number -> the field matrix row of its start (text) or value (integer)
_TEXT = {0: nv.SAM_F_NAME_START, 2: nv.SAM_F_RNAME_START, 5: nv.SAM_F_CIGAR_START, 6: nv.SAM_F_RNEXT_START,
         9: nv.SAM_F_SEQ_START, 10: nv.SAM_F_QUAL_START, 11: nv.SAM_F_EXTRA_START}
_INT = {1: nv.SAM_F_FLAG, 3: nv.SAM_F_POS, 4: nv.SAM_F_MAPQ, 7: nv.SAM_F_PNEXT, 8: nv.SAM_F_TLEN}


def raise_fault(st, line_offset=0):
    """FormatException for the first column or CIGAR fault of a ScanStatus, if it holds one."""
    fault = st.column_fault()
    if fault is not None:
        line, col, kind = fault
        raise FormatException(f"{_FAULTS.get(kind, 'Invalid line')} (column {col})", line_number=line + line_offset)


class SAMBuffer(DelimitedBuffer):
    """SAMBuffer (io/buffers/sam.py): the 11 mandatory SAM columns and the rest of the line (SAMEntry).  Read only."""
    COMMENT = "@"
    dataclass = SAMEntry

    def __init__(self, data, n_lines, fields):
        super().__init__(data, n_lines, None)
        self._f = fields                        # int64[SAM_FIELDS, n_lines] (bnpk_sam_columns)
        self._cache = {}

    @classmethod
    def from_raw_buffer(cls, chunk, header_data=None):
        chunk = _to_device_bytes(chunk)
        n_lines = ops.count_byte(chunk, 10) if chunk.numel() else 0
        if n_lines == 0:
            raise IncompleteEntryException("No complete line in the buffer. Try increasing chunk_size.")
        starts, lens, _ = ops.line_split(chunk, 1, 0, 0, ord(cls.COMMENT), False, 0, max_rows=n_lines)
        fields, status = ops.sam_columns(chunk, starts, lens)
        return cls._from_fields(chunk, n_lines, fields, status, starts[-1:] + lens[-1:])

    @classmethod
    def _from_fields(cls, chunk, n_lines, fields, status, last_end):
        st, end = ops.read_back(status, last_end)          # the one synchronisation of the columns
        raise_fault(st)
        return cls(chunk[:end + 1], n_lines, fields)

    def _text(self, row):
        return FieldView(self._data, self._f[row + 1], self._f[row])

    def get_field_by_number(self, i, t=None):
        if i not in self._cache:
            if i in _TEXT:
                self._cache[i] = self._text(_TEXT[i])
            elif i in _INT:
                self._cache[i] = self._f[_INT[i]]
            else:
                raise IndexError(i)
        return self._cache[i]

    @classmethod
    def formatted(cls, entries):
        raise NotImplementedError("writing SAM is not supported")

    from_data = formatted


class SAMIntervalBuffer(SAMBuffer):
    """The placed alignments of a SAM chunk as Bed6 rows (BamIntervalBuffer for SAM): chromosome, start = POS - 1,
    stop = start + the reference length of its CIGAR (summed on the device; the cigar arrays are never built), name,
    score = MAPQ, strand '-' where flag 0x10 is set.  Records whose RNAME is '*' are left out.  The CIGAR fault and the
    placed-row count are read back with the columns' fault and the chunk's size, in the chunk's one read-back."""
    dataclass = Bed6

    def __init__(self, data, n_lines, fields, ref_len=None, placed=None):
        super().__init__(data, n_lines, fields)
        self._ref_len = ref_len
        self._placed = placed

    @classmethod
    def _from_fields(cls, chunk, n_lines, fields, status, last_end):
        starts, lens = fields[nv.SAM_F_CIGAR_START], fields[nv.SAM_F_CIGAR_LEN].to(torch.int32)
        _, ref_len, cigar_status = ops.cigar_count(chunk, starts, lens)
        rname, rname_len = fields[nv.SAM_F_RNAME_START], fields[nv.SAM_F_RNAME_LEN]
        placed = ((rname_len != 1) | (chunk[rname] != ord("*"))).to(torch.uint8)
        st, cigar_st, n_placed, end = ops.read_back(status, cigar_status, placed.sum(), last_end)
        raise_fault(st)
        raise_fault(cigar_st)
        idx = torch.nonzero_static(placed, size=n_placed).reshape(-1)
        return cls(chunk[:end + 1], n_lines, fields, ref_len, idx)

    def count_entries(self) -> int:
        return self._placed.numel()

    def __len__(self):
        return self.count_entries()

    def _row(self, f):
        return self._f[f][self._placed]

    def get_field_by_number(self, i, t=None):
        if i not in self._cache:
            if i in (0, 3):
                row = nv.SAM_F_RNAME_START if i == 0 else nv.SAM_F_NAME_START
                v = FieldView(self._data, self._row(row + 1), self._row(row))
            elif i == 1:
                v = self._row(nv.SAM_F_POS) - 1
            elif i == 2:
                v = self._row(nv.SAM_F_POS) - 1 + self._ref_len[self._placed]
            elif i == 4:
                v = self._row(nv.SAM_F_MAPQ)
            elif i == 5:
                v = EncodedArray(((self._row(nv.SAM_F_FLAG) & 16) != 0).to(torch.uint8), StrandEncoding)
            else:
                raise IndexError(i)
            self._cache[i] = v
        return self._cache[i]
