"""Alignments (mirror of bionumpy/alignments/__init__.py:9-32 and alignments/cigar.py:18-24)."""
import torch

from .. import ops
from ..datatypes import Bed6, SAMEntry
from ..encoded_array import EncodedArray, EncodedRaggedArray, as_encoded_array
from ..encodings import CigarOpEncoding, StrandEncoding
from ..ragged import RaggedArray
from ..streams import streamable

# M (0), D (2), N (3), = (7) and X (8): the cigar ops that consume the reference
_CONSUMING = sum(1 << op for op in (0, 2, 3, 7, 8))


def count_reference_length(cigar_op, cigar_length):
    """cigar.py:18-24: int64 per row, the summed lengths of the row's M, D, N, = and X ops."""
    codes = cigar_op.ravel().raw().to(torch.int64)
    consumed = cigar_length.ravel().to(torch.int64) * ((_CONSUMING >> codes) & 1)
    return RaggedArray(consumed, cigar_length.lengths).sum(axis=-1)


def _cigar_rows(cigar_text):
    """The RowView of CIGAR text (a text EncodedRaggedArray such as SAMEntry.cigar, or a list of strings)."""
    from ..rows import RowView
    if not isinstance(cigar_text, EncodedRaggedArray):
        cigar_text = as_encoded_array(cigar_text)
    return RowView(cigar_text)


def _raise_cigar_fault(st):
    from ..io.sam import raise_fault
    raise_fault(st)


def parse_cigar(cigar_text):
    """The ops of every row of SAM CIGAR text, as (EncodedRaggedArray of CigarOpEncoding codes, RaggedArray of int64
    lengths): the types of BamEntry.cigar_op and cigar_length.  "*" has no ops.  A row that is not "*" or ops of 1 to 9
    digits and one of MIDNSHP=X raises FormatException with line_number = the row.  One synchronisation, for the fault
    and the total op count."""
    rows = _cigar_rows(cigar_text)
    counts, _, status = ops.cigar_count(rows.base, rows.starts, rows.lens)
    offsets = ops.row_offsets(counts)
    st, total = ops.read_back(status, offsets[-1:])
    _raise_cigar_fault(st)
    op, length = ops.cigar_unpack(rows.base, rows.starts, rows.lens, offsets, total)
    return EncodedRaggedArray(EncodedArray(op, CigarOpEncoding), counts), RaggedArray(length, counts)


def _sam_reference_length(alignment):
    rows = _cigar_rows(alignment.cigar)
    _, ref_len, status = ops.cigar_count(rows.base, rows.starts, rows.lens)
    _raise_cigar_fault(ops.read_back(status)[0])
    return ref_len


@streamable()
def alignment_to_interval(alignment) -> Bed6:
    """The stranded interval each alignment covers on its contig (alignments/__init__.py:9-32): start = position,
    stop = position + the reference length of its cigar, name, score = mapq, strand '-' where flag 0x10 is set.  A
    record whose refID is -1 keeps its chromosome "*".  A SAMEntry's position is 1-based: its start is position - 1,
    and its CIGAR text is parsed on the device (an invalid CIGAR raises FormatException naming the row)."""
    strand = EncodedArray(((alignment.flag & 16) != 0).to(torch.uint8), StrandEncoding)
    if isinstance(alignment, SAMEntry):
        start = alignment.position - 1
        return Bed6(alignment.chromosome, start, start + _sam_reference_length(alignment), alignment.name,
                    alignment.mapq, strand)
    length = count_reference_length(alignment.cigar_op, alignment.cigar_length)
    return Bed6(alignment.chromosome, alignment.position, alignment.position + length, alignment.name, alignment.mapq,
                strand)
