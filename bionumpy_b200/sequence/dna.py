"""complement / get_reverse_complement (mirror of bionumpy/sequence/dna.py:10-65) and, as an EXTENSION, canonical
k-mers (min of a k-mer's hash and the hash of its reverse complement -- what `jellyfish count --canonical` counts,
benchmarks/rules/kmer_counting.smk:11; the reference itself has no such function).

The complement is the reference's 256-entry Lookup for the array's encoding: for an AlphabetEncoding the code of the
complementary letter, for BaseEncoding (ASCII text) the table that knows A, C, G, T, N in upper case and maps every
other byte to 0 (dna.py:29-34).  Reversing the rows and looking the bytes up happen in one kernel
(bnpk_rows_reverse_complement)."""
import numpy as np
import torch

from .. import _native as nv
from .. import ops
from ..encoded_array import EncodedArray, EncodedRaggedArray, as_encoded_array
from ..encodings.alphabet_encoding import AlphabetEncoding
from ..rows import RowView
from ..streams import streamable

_complements = {"A": "T", "G": "C", "C": "G", "T": "A", "N": "N"}
_lut_cache = {}


def _complement_table(encoding) -> np.ndarray:
    """dna.py:13-34 as a 256-entry uint8 table over raw values (codes or ASCII bytes)."""
    table = np.zeros(256, dtype=np.uint8)
    if isinstance(encoding, AlphabetEncoding):
        alphabet = encoding.get_alphabet()
        for i, c in enumerate(alphabet):
            table[i] = alphabet.index(_complements[c])      # KeyError/ValueError like the reference for non-DNA alphabets
        return table
    if encoding.is_base_encoding():
        for key, value in _complements.items():
            table[ord(key)] = ord(value)
        return table
    raise ValueError(f"Invalid encoding for dna-complement: {encoding}")


def _device_table(encoding, device):
    key = (repr(encoding), device.type, device.index)
    if key not in _lut_cache:
        _lut_cache[key] = torch.from_numpy(_complement_table(encoding)).to(device)
    return _lut_cache[key]


def complement(_array):
    """dna.py:36-46: element-wise complement, same shape."""
    array = _array.ravel() if isinstance(_array, EncodedRaggedArray) else _array
    assert isinstance(array, EncodedArray)
    raw = array.raw()
    if not raw.is_cuda:
        raise nv.NativeLibraryError("complement needs a CUDA tensor: bionumpy_b200 has no CPU fallback")
    new = _device_table(array.encoding, raw.device)[raw.to(torch.int64)]
    out = EncodedArray(new.reshape(raw.shape), array.encoding)
    if isinstance(_array, EncodedRaggedArray):
        return EncodedRaggedArray(out, _array._lens)
    return out


@streamable()
def get_reverse_complement(sequence):
    """dna.py:49-65: complement(sequence)[..., ::-1] -- every row reversed and complemented, in one pass."""
    if hasattr(sequence, "sequence") and not isinstance(sequence, (EncodedArray, EncodedRaggedArray)):
        # @apply_to_npdataclass("sequence") (dna.py:50): a record chunk gets its sequence field replaced
        import copy
        out = copy.copy(sequence)
        out.sequence = get_reverse_complement(sequence.sequence)
        return out
    sequence = as_encoded_array(sequence)
    if isinstance(sequence, EncodedArray):
        assert sequence.ndim == 1, "only 1-D EncodedArray and EncodedRaggedArray are supported"
    rows = RowView(sequence)
    lut = _device_table(sequence.encoding, rows.base.device)
    out, _ = ops.rows_reverse_complement(rows.base, rows.starts, rows.lens, lut)
    if rows.flat:
        return EncodedArray(out, sequence.encoding)
    return EncodedRaggedArray(EncodedArray(out, sequence.encoding), rows.lens)


def _interval_sequences(sequence, intervals, stranded):
    """sequence[intervals.start:intervals.stop] row by row (dna.py:68-106), a '-' row reverse-complemented when
    ``stranded``: bnpk_interval_gather in flat mode, one synchronisation for the output size."""
    sequence = as_encoded_array(sequence)
    assert isinstance(sequence, EncodedArray) and sequence.ndim == 1, "intervals index one 1-D sequence"
    raw = sequence.raw()
    if not raw.is_cuda:
        raise nv.NativeLibraryError("interval sequences need a CUDA tensor: bionumpy_b200 has no CPU fallback")
    raw = raw.to(torch.uint8).contiguous()
    start, stop = (torch.as_tensor(v).to(raw.device, torch.int64).contiguous() for v in (intervals.start, intervals.stop))
    strand = lut = None
    if stranded:
        from ..encodings import StrandEncoding
        s = intervals.strand
        minus = 1 if getattr(s, "encoding", None) == StrandEncoding else ord("-")
        strand = (torch.as_tensor(s.raw() if hasattr(s, "raw") else s).reshape(-1).to(raw.device) == minus)
        strand = strand.to(torch.uint8).contiguous()
        lut = _device_table(sequence.encoding, raw.device)
    out, row_lens, bad, _ = ops.interval_gather(raw, start, stop, strand=strand, complement_lut=lut)
    if bad is not None:
        raise ValueError(f"interval {bad} ({int(start[bad])}-{int(stop[bad])}) is not inside the sequence "
                         f"({raw.numel()} bases)")
    return EncodedRaggedArray(EncodedArray(out, sequence.encoding), row_lens)


@streamable()
def get_strand_specific_sequences(encoded_array, stranded_intervals) -> EncodedRaggedArray:
    """dna.py:68-88: the sequence of every interval, reverse-complemented where its strand is '-' (the complement of
    the sequence's encoding: for ASCII text A, C, G, T, N, every other byte 0)."""
    return _interval_sequences(encoded_array, stranded_intervals, True)


@streamable()
def get_sequences(sequence, intervals) -> EncodedRaggedArray:
    """dna.py:91-106: the sequence of every interval, strands ignored."""
    return _interval_sequences(sequence, intervals, False)


def complement_xor_of(alphabet_encoding) -> int:
    """The complement of a four-letter DNA/RNA alphabet as an XOR on the 2-bit code (3 for ACGT order, 2 for ACTG /
    ACUG order); raises for alphabets where it is not an XOR."""
    letters = [c.replace("U", "T") for c in alphabet_encoding.get_alphabet()]
    assert len(letters) == 4, "canonical k-mers need a four-letter alphabet"
    comp = [letters.index(_complements[c]) for c in letters]
    x = comp[0]
    assert all((i ^ x) == c for i, c in enumerate(comp)), "complement is not an XOR for this alphabet order"
    return x
