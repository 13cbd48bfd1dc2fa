"""Alignments (mirror of bionumpy/alignments/__init__.py:9-32 and alignments/cigar.py:18-24)."""
import torch

from ..datatypes import Bed6
from ..encoded_array import EncodedArray
from ..encodings import StrandEncoding
from ..ragged import RaggedArray
from ..streams import streamable

# M (0), D (2), N (3), = (7) and X (8): the cigar ops that consume the reference
_CONSUMING = sum(1 << op for op in (0, 2, 3, 7, 8))


def count_reference_length(cigar_op, cigar_length):
    """cigar.py:18-24: int64 per row, the summed lengths of the row's M, D, N, = and X ops."""
    codes = cigar_op.ravel().raw().to(torch.int64)
    consumed = cigar_length.ravel().to(torch.int64) * ((_CONSUMING >> codes) & 1)
    return RaggedArray(consumed, cigar_length.lengths).sum(axis=-1)


@streamable()
def alignment_to_interval(alignment) -> Bed6:
    """The stranded interval each alignment covers on its contig (alignments/__init__.py:9-32): start = position,
    stop = position + the reference length of its cigar, name, score = mapq, strand '-' where flag 0x10 is set.  A
    record whose refID is -1 keeps its chromosome "*"."""
    strand = EncodedArray(((alignment.flag & 16) != 0).to(torch.uint8), StrandEncoding)
    length = count_reference_length(alignment.cigar_op, alignment.cigar_length)
    return Bed6(alignment.chromosome, alignment.position, alignment.position + length, alignment.name, alignment.mapq,
                strand)
