"""Position weight matrices: PWM, PositionWeightMatrix, get_motif_scores (mirror of
bionumpy/sequence/position_weight_matrix.py:13-196).

The matrix is built on the host with NumPy float64 by the reference's expressions, so it has the reference's bits.
Every score is computed on the GPU by the motif kernels (K7, include/bnpk.h bnpk_rows_pwm_scores / bnpk_rows_pwm_max):
each position's score is +0.0 plus the matrix entries of its bases added one column at a time, in column order, in
float64 -- the reference's own sequence of adds (calculate_scores, :96-99), so the scores are the reference's bits.
``get_motif_scores`` on ragged sequences returns a lazy float64 RaggedArray: ``.max(axis=-1)`` before first use runs the
fused kernel and never writes the scores.  There is no CPU fallback."""
import typing
from typing import Dict

import numpy as np
import torch

from .. import config, ops
from ..encoded_array import EncodedArray, EncodedRaggedArray, as_encoded_array
from ..encodings.alphabet_encoding import AlphabetEncoding
from ..ragged import LazyRaggedArray, segment_max
from ..rows import RowView

MAX_MOTIF_LEN = 1024          # the row kernels' segment overlap
MAX_TABLE_CELLS = 8192        # alphabet_size * motif length doubles: 64 KiB of shared memory


def _pwm_from_counts(count_matrix):
    """position_weight_matrix.py:26-28."""
    with_pseudo = count_matrix + 1
    return np.log(with_pseudo / with_pseudo.sum(axis=0, keepdims=True))


class PWM:
    """A position weight matrix: log-likelihood ratios of the motif against a background (position_weight_matrix.py:
    31-140).  ``matrix`` is float64 [len(alphabet), motif length]."""

    def __init__(self, matrix, alphabet):
        self._matrix = matrix
        self._alphabet = alphabet
        self._encoding = AlphabetEncoding(alphabet)
        self._indices = np.arange(self.window_size)
        self._dev_matrix = {}

    @property
    def alphabet(self) -> str:
        return self._alphabet

    @property
    def window_size(self) -> int:
        return self._matrix.shape[-1]

    def __str__(self):
        matrix = self._matrix.transpose()
        return "PWM with alphabet " + self._alphabet + "\n" + \
               '\n'.join([' '.join([str(round(c, 2)) for c in row]) for row in matrix])

    @classmethod
    def from_dict(cls, dictionary: Dict[str, typing.Union[np.ndarray, typing.List]],
                  background: Dict[str, float] = None) -> "PWM":
        """Log-likelihood ratios log(p) - log(background) from position probabilities (uniform background by default),
        position_weight_matrix.py:102-130."""
        if background is None:
            background = {key: 1 / len(dictionary) for key in dictionary}
        alphabet = "".join(dictionary.keys())
        with np.errstate(divide="ignore"):
            matrix = np.log(np.array(list(dictionary.values()))) - \
                np.log([background[key] for key in dictionary])[:, np.newaxis]
        return cls(matrix, alphabet)

    @classmethod
    def from_counts(cls, counts: Dict[str, typing.List[int]]) -> "PWM":
        """log((c + 1) / column sum of (c + 1)), position_weight_matrix.py:132-135."""
        return cls(_pwm_from_counts(np.array(list(counts.values()))), "".join(counts.keys()))

    # -- device plumbing ----------------------------------------------------------------------
    def _check_limits(self):
        m, a = self.window_size, len(self._alphabet)
        if not 1 <= m <= MAX_MOTIF_LEN:
            raise ValueError(f"motif length {m} is outside 1..{MAX_MOTIF_LEN}")
        if not 2 <= a <= 255 or a * m > MAX_TABLE_CELLS:
            raise ValueError(f"alphabet size {a} times motif length {m} must be at most {MAX_TABLE_CELLS}, "
                             "with 2..255 letters")

    def device_matrix(self, device):
        """[motif length, alphabet size] float64 on ``device``: the transpose of ``_matrix``, one column contiguous."""
        key = (device.type, device.index)
        if key not in self._dev_matrix:
            t = np.ascontiguousarray(np.asarray(self._matrix, dtype=np.float64).T)
            self._dev_matrix[key] = torch.from_numpy(t).to(device)
        return self._dev_matrix[key]

    def _rows(self, sequence) -> RowView:
        """as_valid_encoded_array (position_weight_matrix.py:45-55) as a kernel input: text is read with
        AlphabetEncoding(alphabet); an AlphabetEncoding array is read as codes when its alphabet starts with this one
        and every code is below len(alphabet)."""
        self._check_limits()
        if isinstance(sequence, (str, list, np.ndarray)):
            sequence = as_encoded_array(sequence)
        if not isinstance(sequence, (EncodedArray, EncodedRaggedArray)):
            raise TypeError(f"cannot score {type(sequence)}")
        rows = RowView(sequence, self._encoding)
        enc = sequence.encoding
        if enc.is_base_encoding():
            return rows
        if isinstance(enc, AlphabetEncoding):
            alphabet = list(enc.get_alphabet())
            s_alphabet = list(self._alphabet)
            codes = sequence.ravel().raw() if isinstance(sequence, EncodedRaggedArray) else sequence.raw()
            top = int(codes.max().item()) if codes.numel() else 0
            if not alphabet[:len(self._alphabet)] == s_alphabet or top >= len(self._alphabet):
                raise Exception(f'Could not calculate pwm for alphabet {s_alphabet} on {alphabet} encoded array')
            return rows
        as_encoded_array(sequence, self._encoding)          # raises the reference's EncodingException
        raise TypeError(f"cannot score an array encoded with {enc}")

    def _rescan(self, rows: RowView):
        """The status of the fused maximum on the rows themselves: it places a bad base that a launch on pieces of
        the rows reported (error path)."""
        return ops.rows_pwm_max(rows.base, rows.starts, rows.lens, rows.enc_mode, self.device_matrix(rows.base.device),
                                rows.lut)[1]

    def _window_scores(self, rows: RowView):
        """The scores of every window of every row, flat float64.  Long rows are cut into overlapping pieces, one warp
        each."""
        m = self.window_size
        mat = self.device_matrix(rows.base.device)
        p, offsets, total, piece_row = rows.split(m, ops.row_offsets(rows.lens, m - 1))
        scores, _, status = ops.rows_pwm_scores(rows.base, p.starts, p.lens, rows.enc_mode, mat, rows.lut,
                                                offsets=offsets, total=total)
        rows.raise_bad_base(status, self._rescan if piece_row is not None else None)
        return scores

    def _row_max(self, rows: RowView):
        """max(axis=-1) of the window scores of every row without writing them: NaN-propagating, -inf for a row
        without a window.  The pieces of a long row are combined on the device."""
        mat = self.device_matrix(rows.base.device)
        p, _, _, piece_row = rows.split(self.window_size)
        best, status = ops.rows_pwm_max(rows.base, p.starts, p.lens, rows.enc_mode, mat, rows.lut)
        rows.raise_bad_base(status, self._rescan if piece_row is not None else None)
        if piece_row is not None:
            best = segment_max(best, piece_row, rows.lens.numel())
        return best

    # -- scoring ------------------------------------------------------------------------------
    def calculate_score(self, sequence) -> float:
        """The score of a sequence as long as the motif (position_weight_matrix.py:66-79); for a 2-D array, one score
        per row.  Computed on the GPU in column order; the reference sums with NumPy's pairwise ``.sum(axis=-1)``,
        which for motifs of 8 or more columns can differ from it in the last bits (relative 1e-12)."""
        rows = self._rows(sequence)
        if bool((rows.lens != self.window_size).any().item()):
            raise AssertionError(f"sequence length must be the motif length {self.window_size}")
        scores = self._window_scores(rows)
        return scores[0].item() if rows.flat else scores

    def calculate_scores(self, sequence) -> torch.Tensor:
        """Scores of every position of the flattened sequence (position_weight_matrix.py:83-100): the last m - 1
        positions hold the sums of the columns that fit.  float64 tensor of the sequence's size."""
        if isinstance(sequence, list):
            sequence = as_encoded_array(sequence)
        if isinstance(sequence, EncodedRaggedArray) or (isinstance(sequence, EncodedArray) and sequence.ndim > 1):
            sequence = sequence.ravel()
        rows = self._rows(sequence)
        m = self.window_size
        scores = self._window_scores(rows)             # validates every byte, the last m - 1 included
        L = int(rows.lens[0].item())
        tail_start = max(L - (m - 1), 0)
        if tail_start == L:
            return scores
        # the last m - 1 positions: one short row scored with the columns that fit
        t_lens = torch.full((1,), L - tail_start, dtype=torch.int32, device=rows.base.device)
        tail, _, _ = ops.rows_pwm_scores(rows.base, rows.starts + tail_start, t_lens, rows.enc_mode,
                                         self.device_matrix(rows.base.device), rows.lut, tail=True)
        return torch.cat([scores[:tail_start], tail])


class LazyMotifScores(LazyRaggedArray):
    """float64 RaggedArray of the window scores of every row, computed on first use; ``max(axis=-1)`` before that runs
    the fused maximum instead."""

    def __init__(self, pwm: PWM, rows: RowView):
        self._pwm, self._rows = pwm, rows
        super().__init__(rows.lens, pwm.window_size - 1)

    def _compute(self):
        return self._pwm._window_scores(self._rows)

    def max(self, axis=None, **kwargs):
        if axis in (-1, 1) and not self.is_materialised():
            return self._pwm._row_max(self._rows)
        return super().max(axis=axis, **kwargs)


class PositionWeightMatrix:
    """The PWM as a rolling function (position_weight_matrix.py:13-23, sequence/rollable.py:30-80)."""

    def __init__(self, pwm: PWM):
        self._pwm = pwm
        self._encoding = pwm._encoding
        self.window_size = pwm.window_size

    def __call__(self, sequence) -> float:
        return self._pwm.calculate_score(sequence)

    def rolling_window(self, sequence, window_size: int = None, mode: str = "valid"):
        """The score of every window of the sequence(s): what get_motif_scores returns."""
        assert window_size in (None, self.window_size) and mode == "valid", "only the motif's own valid windows"
        return get_motif_scores(sequence, self._pwm)


def get_motif_scores(sequence, pwm: PWM):
    """Motif scores of every window of every row (position_weight_matrix.py:166-196): a float64 RaggedArray with
    max(L - m + 1, 0) scores per row of length L, or for a 1-D sequence a float64 tensor of N - m + 1 scores.

    A one-column PWM gives one score per base, as ``PositionWeightMatrix.rolling_window`` does in the reference (its
    ``get_motif_scores`` returns empty rows there).  The ragged result is lazy: ``.max(axis=-1)`` on it before first use
    computes the per-row maximum without writing the scores.

    >>> pwm = PWM.from_dict({"A": [5, 1], "C": [1, 5], "G": [0, 0], "T": [0, 0]})
    >>> get_motif_scores(["ACTGAC", "CA", "GG"], pwm).tolist()
    [[5.991464547107982, -inf, -inf, -inf, 5.991464547107982], [2.772588722239781], [-inf]]
    """
    rows = pwm._rows(sequence)
    if rows.flat:
        return pwm._window_scores(rows)
    out = LazyMotifScores(pwm, rows)
    if not config.LAZY:
        out._data
    return out
