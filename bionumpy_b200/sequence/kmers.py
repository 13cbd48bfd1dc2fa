"""get_kmers / count_kmers (mirror of bionumpy/sequence/kmers.py:36-145).

Hash definition (pinned against the reference's doc goldens): h = sum_j code[i+j] * 4^j, int64,
per-row windows only, rows shorter than k give empty rows.  ``get_kmers`` returns a lazily
materialised EncodedRaggedArray: asking for ``.raw()``/indexing runs the hash kernel (K3);
``count_encoded(kmers, axis=None)`` runs the fused hash+histogram kernel instead and never
writes the hashes."""
import logging

import torch

from .. import config, ops
from ..encoded_array import EncodedArray, EncodedRaggedArray
from ..encodings.alphabet_encoding import AlphabetEncoding, DNAEncoding
from ..encodings.exceptions import EncodingError
from ..encodings.kmer_encodings import KmerEncoding
from ..ragged import LazyRaggedArray
from ..rows import LONG_ROW, RowView, _split_long_rows  # noqa: F401 (the split is also imported from here)
from ..streams import streamable
from .count_encoded import count_encoded, count_hashed, EncodedCounts

logger = logging.getLogger(__name__)


def _source_of(sequence) -> RowView:
    """The rows k-mers are taken from: text is read as DNAEncoding (kmers.py:70-72), encoded arrays need an
    AlphabetEncoding."""
    if isinstance(sequence, EncodedArray):
        assert sequence.ndim == 1, "only 1-D EncodedArray and EncodedRaggedArray are supported"
    rows = RowView(sequence, DNAEncoding)
    assert isinstance(rows.alphabet_encoding, AlphabetEncoding), \
        "Sequence needs to be encoded with an AlphabetEncoding, e.g. DNAEncoding. " \
        "Change encoding of your sequences by using e.g. bnp.change_encoding(sequences, bnp.DNAEncoding)"
    return rows


def rescan_kmers(rows: RowView):
    """The status of counting the rows' 1-mers: it reads every byte, so it places a bad base that a launch on pieces
    or batches of the rows reported (error path)."""
    return ops.rows_kmer_count(rows.base, rows.starts, rows.lens, rows.enc_mode, 1, 4, 0, rows.lut)[1]


class LazyKmerValues(LazyRaggedArray, EncodedRaggedArray):
    """EncodedRaggedArray of k-mer hashes / minimizers whose int64 data appear on first use."""

    def __init__(self, rows: RowView, k: int, window_size: int, canonical: bool = False):
        self._rows, self._k, self._window = rows, k, window_size
        self._canonical = canonical
        if canonical:
            from .dna import complement_xor_of
            assert window_size == 0, "canonical minimizers are not implemented"
            self._cxor = complement_xor_of(rows.alphabet_encoding)
        super().__init__(rows.lens, (window_size if window_size else k) - 1)
        self._encoding = KmerEncoding(rows.alphabet_encoding, k)

    def _compute(self):
        s = self._rows
        if s.alphabet_encoding.alphabet_size != 4:
            # the reference's generic dot-product path (kmers.py:87): plain k-mers only
            if self._window:
                raise NotImplementedError("minimizers are only implemented for 4-letter alphabets")
            vals, _, status = ops.rows_generic_hash(s.base, s.starts, s.lens, s.alphabet_encoding.alphabet_size, self._k, None)
            return vals
        span = self._window if self._window else self._k
        p, offsets, total, piece_row = s.split(span, ops.row_offsets(s.lens, span - 1))
        if self._window:
            vals, _, status = ops.rows_minimizers(s.base, p.starts, p.lens, s.enc_mode, self._k, self._window, s.lut,
                                                  offsets, total=total)
        elif self._canonical:
            vals, _, status = ops.rows_kmer_hash_canonical(s.base, p.starts, p.lens, s.enc_mode, self._k, self._cxor,
                                                           s.lut, offsets, total=total)
        else:
            vals, _, status = ops.rows_kmer_hash(s.base, p.starts, p.lens, s.enc_mode, self._k, s.lut, offsets,
                                                 total=total)
        self._check(status, split=piece_row is not None)
        return vals

    def _check(self, status, split=False):
        try:
            self._rows.raise_bad_base(status, rescan_kmers if split else None)
        except EncodingError:
            logging.error("Tried to change encoding of sequences to DNAEncoding, but failed. "
                          "Make sure your sequences are valid DNA, only containing A, C, G, and T")
            raise

    def fused_histogram(self, n_bins: int) -> torch.Tensor:
        """hist[b] = #{values == b (mod n_bins)} without writing the values (K3/K4 + K5 fused)."""
        s = self._rows
        if s.alphabet_encoding.alphabet_size != 4:
            hist, _ = ops.bincount(self._data.contiguous(), n_bins)
            return hist
        if self._canonical:
            hist, status = ops.rows_kmer_count_canonical(s.base, s.starts, s.lens, s.enc_mode, self._k, self._cxor, n_bins, s.lut)
            self._check(status)
            return hist
        buf = s.chunk_buffer
        if buf is not None and buf.can_fuse_count():
            return buf.fused_kmer_histogram(self._k, self._window, n_bins, s)
        p, _, _, piece_row = s.split(self._window if self._window else self._k)
        hist, status = ops.rows_kmer_count(s.base, p.starts, p.lens, s.enc_mode, self._k, n_bins, self._window, s.lut)
        self._check(status, split=piece_row is not None)
        return hist


def get_kmers(sequence, k: int, canonical: bool = False):
    """kmers.py:36-87.  ``sequence``: EncodedRaggedArray / 1-D EncodedArray, BaseEncoding text or an
    AlphabetEncoding with four letters; k in 1..31.  EXTENSION: ``canonical=True`` gives min(hash, hash of the
    reverse complement) for every k-mer (sequence/dna.py)."""
    assert 0 < k < 32, "k must be larger than 0 and smaller than 32"
    out = LazyKmerValues(_source_of(sequence), k, 0, canonical=canonical)
    if not config.LAZY:
        out._data
    if isinstance(sequence, EncodedArray):
        return EncodedArray(out._data, out.encoding)
    return out


@streamable(sum)
def count_kmers(sequence, k: int, axis=None) -> EncodedCounts:
    """kmers.py:129-145."""
    return count_encoded(get_kmers(sequence, k), axis=axis)


def count_kmers_hashed(sequence, k: int, n_buckets: int = 1 << 24, window_size: int = 0, canonical: bool = False) -> torch.Tensor:
    """EXTENSION: np.bincount(get_kmers(sequence, k) % n_buckets) (or of the minimizers when
    window_size > 0) as an int64 CUDA tensor, fused."""
    assert 0 < k < 32, "k must be larger than 0 and smaller than 32"
    assert window_size == 0 or k <= window_size, "kmer size must be smaller than window size"
    return count_hashed(LazyKmerValues(_source_of(sequence), k, window_size, canonical=canonical), n_buckets)
