"""AlphabetEncoding (mirror of bionumpy/encodings/alphabet_encoding.py:8-107).

The byte -> code map is the reference's 256-entry LUT (255 = invalid, case-insensitive).  On the
device the two DNA alphabets are closed-form bit tricks (BNPK_ENC_ASCII_ACGT / _ACTG); every other
alphabet ships its LUT to the kernel (BNPK_ENC_LUT)."""
from typing import List

import numpy as np
import torch

from .. import _native as nv
from ..encoded_array import OneToOneEncoding, EncodedArray, EncodedRaggedArray, BaseEncoding
from .exceptions import EncodingError


class AlphabetEncoding(OneToOneEncoding):
    def __init__(self, alphabet: str):
        self._raw_alphabet = [c.upper() for c in alphabet]
        self._alphabet_size = len(self._raw_alphabet)
        self._alphabet = np.array([ord(c) for c in self._raw_alphabet], dtype=np.uint8)
        lower = self._alphabet + (ord("a") - ord("A"))
        self._lookup = np.full(256, 255, dtype=np.uint8)          # alphabet_encoding.py:19-32
        self._lookup[self._alphabet] = np.arange(self._alphabet_size)
        self._lookup[lower] = np.arange(self._alphabet_size)
        self._dev_luts = {}

    # -- device plumbing ----------------------------------------------------------------------
    @property
    def enc_mode(self) -> int:
        """How the kernels should read ASCII text into this alphabet."""
        letters = "".join(self._raw_alphabet)
        if letters == "ACGT":
            return nv.ENC_ASCII_ACGT
        if letters == "ACTG":
            return nv.ENC_ASCII_ACTG
        return nv.ENC_LUT

    def device_lut(self, device):
        key = (device.type, device.index)
        if key not in self._dev_luts:
            self._dev_luts[key] = torch.from_numpy(self._lookup.copy()).to(device)
        return self._dev_luts[key]

    def _raise_encoding_error(self, offset):
        """alphabet_encoding.py:37-46: offset = first invalid index of the flattened array."""
        raise EncodingError(f"Error when encoding to {self.__class__.__name__}({''.join(self._raw_alphabet)}). "
                            f"Invalid character at flat offset {offset}", offset)

    def _encode_rows(self, rows):
        from .. import ops
        codes, _, status = ops.rows_encode(rows.base, rows.starts, rows.lens, rows.enc_mode, rows.lut)
        rows.raise_bad_base(status)
        return codes

    def _encode(self, byte_tensor):
        """Flat bytes -> codes (alphabet_encoding.py:34-46), as one row."""
        from ..rows import RowView
        rows = RowView(EncodedArray(byte_tensor.reshape(-1), BaseEncoding), self)
        return self._encode_rows(rows).reshape(byte_tensor.shape)

    def _encode_ragged(self, ragged):
        """Encode a (base, starts, lens) view straight from the raw chunk -- no gather pass."""
        from ..rows import RowView
        rows = RowView(ragged, self)
        return EncodedRaggedArray(EncodedArray(self._encode_rows(rows), self), rows.lens)

    def _decode(self, encoded):
        alpha = torch.from_numpy(self._alphabet).to(encoded.device)
        return alpha[encoded.to(torch.int64)]

    # -- reference surface ------------------------------------------------------------------------
    @property
    def alphabet_size(self) -> int:
        return self._alphabet_size

    def get_alphabet(self) -> List[str]:
        return [chr(c) for c in self._alphabet]

    def get_labels(self) -> List[str]:
        return self.get_alphabet()

    def __str__(self):
        return f"""AlphabetEncoding('{"".join(self.get_alphabet())}')"""

    __repr__ = __str__

    def __eq__(self, other):
        if not isinstance(other, AlphabetEncoding):
            return False
        return len(self._alphabet) == len(other._alphabet) and bool(np.all(self._alphabet == other._alphabet))

    def __hash__(self):
        return hash(repr(self))


ACTGEncoding = AlphabetEncoding("ACTG")
ACGTEncoding = AlphabetEncoding("ACGT")
DNAEncoding = ACGTEncoding
ACUGEncoding = AlphabetEncoding("ACUG")
RNAENcoding = ACUGEncoding
AminoAcidEncoding = AlphabetEncoding('ACDEFGHIKLMNPQRSTVWY*')
StrandEncoding = AlphabetEncoding("+-.")      # alphabet_encoding.py:120: '+' 0, '-' 1, '.' 2
BamEncoding = AlphabetEncoding("=ACMGRSVTWYHKDBN")   # the 4-bit base codes of BAM (SAM spec 4.2.3)
CigarOpEncoding = AlphabetEncoding("MIDNSHP=X")      # the cigar op codes of BAM (SAM spec 4.2.2)
