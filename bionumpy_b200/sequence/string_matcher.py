"""String and pattern matching: match_string, StringMatcher, FixedLenRegexMatcher, RegexMatcher (mirror of
bionumpy/sequence/string_matcher.py).

A pattern is parsed on the host into columns of symbol sets and expanded into sub-patterns, one per combination of gap
lengths.  Every match is computed on the GPU by the match kernels (K8, include/bnpk.h bnpk_rows_match /
bnpk_rows_match_count).  Text is read in the matcher's encoding inside the kernel; a byte outside the alphabet raises
the EncodingError of ``as_encoded_array``.  Ragged results are lazy: ``.sum(axis=-1)``, ``.any(axis=-1)`` and
``.mean(axis=-1)`` before first use run the fused count and never write the matches.  There is no CPU fallback.

Grammar: literal symbols, ``.`` (any symbol), ``[...]`` classes of literal symbols and, for RegexMatcher, gaps
``.{a,b}`` (``a`` may be empty, 0 <= a <= b) with at least one column on each side.  The reference recognises a gap
only after a group of letters or classes; this grammar is a superset of that.  RegexMatcher gives a value at every
position ("same" mode), True where some expansion matches and fits inside the row -- the one deviation from the
reference, whose windows read on into the next row or past the end of the buffer."""
import copy
import itertools
import re

import numpy as np
import torch

from .. import config, ops
from ..encoded_array import EncodedArray, EncodedRaggedArray, as_encoded_array
from ..encodings.alphabet_encoding import AlphabetEncoding
from ..encodings.exceptions import EncodingError
from ..ragged import LazyRaggedArray, segment_sum
from ..rows import RowView

MAX_SUB_LEN = 1024            # columns of one sub-pattern: the row kernels' segment overlap
MAX_SUBS = 64                 # sub-patterns of one expanded pattern
MAX_SET_WORDS = 8192          # columns * ceil(alphabet size / 32) words: 32 KiB of shared memory

_SPECIAL = set("*+?|(){}\\^$[]")
_GAP = re.compile(r"\.\{(\d*),(\d+)\}")


def parse_pattern(pattern: str, literal=False):
    """The columns of ``pattern``: a list whose items are a set of symbols (one column), None (``.``, any symbol) or
    a ``(a, b)`` gap.  ``literal``: every character is its own column.  ValueError outside the grammar."""
    if not isinstance(pattern, str):
        raise TypeError(f"a pattern is a str, not {type(pattern)}")
    if not pattern:
        raise ValueError("empty pattern")
    if literal:
        return [{c} for c in pattern]
    items, i = [], 0
    while i < len(pattern):
        c = pattern[i]
        if c == ".":
            g = _GAP.match(pattern, i)
            if g:
                a, b = int(g.group(1) or 0), int(g.group(2))
                if a > b:
                    raise ValueError(f"gap {g.group(0)}: {a} > {b}")
                if not items or not isinstance(items[-1], (set, type(None))):
                    raise ValueError(f"gap {g.group(0)} needs a column before it")
                items.append((a, b))
                i = g.end()
                continue
            if pattern.startswith(".{", i):
                raise ValueError(f"unsupported repetition at {i} in {pattern!r}: gaps are .{{a,b}}")
            items.append(None)
        elif c == "[":
            end = pattern.find("]", i + 1)
            if end < 0:
                raise ValueError(f"unterminated class in {pattern!r}")
            members = pattern[i + 1:end]
            if not members:
                raise ValueError(f"empty class in {pattern!r}")
            if any(m in "[\\^-" for m in members):
                raise ValueError(f"class {pattern[i:end + 1]!r}: only literal symbols")
            items.append(set(members))
            i = end
        elif c in _SPECIAL:
            raise ValueError(f"{c!r} at {i} in {pattern!r} is outside the pattern grammar")
        else:
            items.append({c})
        i += 1
    if isinstance(items[-1], tuple):
        raise ValueError(f"a gap needs a column after it in {pattern!r}")
    return items


def expand(items):
    """The sub-patterns of parsed columns: one list of columns (set or None) per combination of gap lengths."""
    gaps = [range(g[0], g[1] + 1) for g in items if isinstance(g, tuple)]
    subs = []
    for lengths in itertools.product(*gaps):
        cols, it = [], iter(lengths)
        for item in items:
            cols.extend([None] * next(it) if isinstance(item, tuple) else [item])
        subs.append(cols)
    return subs


class _Pattern:
    """An expanded pattern in one encoding: the sub-patterns' lengths and their column sets as device words."""

    def __init__(self, pattern, encoding, literal=False, gaps=True):
        items = parse_pattern(pattern, literal)
        if not gaps and any(isinstance(g, tuple) for g in items):
            raise ValueError(f"{pattern!r}: gaps need a RegexMatcher")
        if encoding.is_base_encoding():
            self.alphabet_size, codes = 256, {chr(b): b for b in range(256)}
        elif isinstance(encoding, AlphabetEncoding):
            self.alphabet_size = encoding.alphabet_size
            codes = {}
            for ch in {m for item in items if isinstance(item, set) for m in item}:
                code = int(encoding._lookup[ord(ch)]) if ord(ch) < 256 else 255
                if code == 255:
                    raise EncodingError(f"{ch!r} of pattern {pattern!r} is not in {encoding}", pattern.index(ch))
                codes[ch] = code
        else:
            raise TypeError(f"cannot match strings in an array encoded with {encoding}")
        self.encoding = encoding
        subs = expand(items)
        if len(subs) > MAX_SUBS:
            raise ValueError(f"{pattern!r} expands into {len(subs)} sub-patterns, more than {MAX_SUBS}")
        self.sub_lens = [len(s) for s in subs]
        if max(self.sub_lens) > MAX_SUB_LEN:
            raise ValueError(f"{pattern!r} has a sub-pattern of {max(self.sub_lens)} columns, more than {MAX_SUB_LEN}")
        wpc = (self.alphabet_size + 31) // 32
        if sum(self.sub_lens) * wpc > MAX_SET_WORDS:
            raise ValueError(f"{pattern!r}: {sum(self.sub_lens)} columns of {wpc} words exceed {MAX_SET_WORDS} words")
        bits = np.zeros((sum(self.sub_lens), wpc * 32), dtype=bool)
        for c, col in enumerate(col for s in subs for col in s):
            if col is None:
                bits[c, :self.alphabet_size] = True
            else:
                bits[c, [codes[m] for m in col]] = True
        self._words = np.packbits(bits, axis=1, bitorder="little").view("<u4").view(np.int32).reshape(-1)
        self.span = max(self.sub_lens)
        self._dev = {}

    def sets(self, device):
        key = (device.type, device.index)
        if key not in self._dev:
            self._dev[key] = torch.from_numpy(self._words.copy()).to(device)
        return self._dev[key]

    # -- device plumbing ----------------------------------------------------------------------
    def rows(self, sequence) -> RowView:
        """The kernel input of ``sequence``: text is read in this pattern's encoding, an encoded array as its codes."""
        if isinstance(sequence, (str, list, np.ndarray)):
            sequence = as_encoded_array(sequence)
        if not isinstance(sequence, (EncodedArray, EncodedRaggedArray)):
            raise TypeError(f"cannot match in {type(sequence)}")
        enc = sequence.encoding
        if self.encoding.is_base_encoding():
            if not enc.is_base_encoding():
                raise TypeError(f"a raw-text pattern cannot match an array encoded with {enc}")
        elif not enc.is_base_encoding() and enc != self.encoding:
            sequence = as_encoded_array(sequence, self.encoding)     # raises the reference's EncodingException
        rows = RowView(sequence, None if self.encoding.is_base_encoding() else self.encoding)
        if rows.enc_mode is None:                                       # raw bytes are their own codes
            rows.enc_mode = ops.nv.ENC_CODES
        return rows

    def _launch_args(self, rows):
        return rows.enc_mode, self.alphabet_size, self.sets(rows.base.device), self.sub_lens

    def _rescan(self, rows):
        return ops.rows_match_count(rows.base, rows.starts, rows.lens, *self._launch_args(rows), lut=rows.lut)[1]

    def _pieces(self, rows, same, offsets=None):
        """The launches of ``rows`` cut into long-row pieces: [(pieces, same, index of the pieces)] and the pieces'
        offsets.  In "same" mode only the last piece of a row tests the row's last span - 1 positions."""
        p, p_off, total, piece_row = rows.split(self.span, offsets)
        if piece_row is None or not same:
            return [(p, same, None)], p_off, total, piece_row
        last = torch.ones_like(piece_row, dtype=torch.bool)
        last[:-1] = piece_row[1:] != piece_row[:-1]
        groups = []
        for sel, s in ((~last, False), (last, True)):
            idx = torch.nonzero(sel).squeeze(1)
            if idx.numel():
                g = copy.copy(p)
                g.starts, g.lens = p.starts[idx].contiguous(), p.lens[idx].contiguous()
                groups.append((g, s, idx))
        return groups, p_off, total, piece_row

    def matches(self, rows, same):
        """The matches of every row, flat bool (contiguous rows)."""
        offsets = ops.row_offsets(rows.lens, 0 if same else self.span - 1)
        groups, p_off, total, piece_row = self._pieces(rows, same, offsets)
        if total is None:
            total = int(offsets[-1].item())
        out = torch.empty(total, dtype=torch.uint8, device=rows.base.device)
        status = ops.nv.new_status(rows.base.device)
        for g, s, idx in groups:
            g_off = p_off if idx is None else p_off[torch.cat([idx, idx[-1:] + 1])]     # and the end of the last piece
            ops.rows_match(g.base, g.starts, g.lens, *self._launch_args(rows), same=s, lut=rows.lut, offsets=g_off,
                           status=status, out=out)
        rows.raise_bad_base(status, self._rescan if piece_row is not None else None)
        return out.view(torch.bool)

    def counts(self, rows, same):
        """The matches of every row counted without writing them: int64[R].  The pieces of a long row are summed on
        the device."""
        groups, _, _, piece_row = self._pieces(rows, same)
        status = ops.nv.new_status(rows.base.device)
        out = None
        for g, s, idx in groups:
            c, _ = ops.rows_match_count(g.base, g.starts, g.lens, *self._launch_args(rows), same=s, lut=rows.lut,
                                        status=status)
            if piece_row is None:
                out = c
            else:
                rows_of = piece_row if idx is None else piece_row[idx]
                part = segment_sum(c, rows_of, rows.lens.numel())
                out = part if out is None else out + part
        rows.raise_bad_base(status, self._rescan if piece_row is not None else None)
        return out


class LazyMatches(LazyRaggedArray):
    """bool RaggedArray of the matches of every row, computed on first use; ``sum``, ``any`` and ``mean`` along
    axis=-1 before that run the fused count instead."""

    def __init__(self, pattern: _Pattern, rows: RowView, same: bool):
        self._pattern, self._rows, self._same = pattern, rows, same
        super().__init__(rows.lens, 0 if same else pattern.span - 1)

    def _compute(self):
        return self._pattern.matches(self._rows, self._same)

    def _fused(self, axis):
        return axis in (-1, 1) and not self.is_materialised()

    def sum(self, axis=None, **kwargs):
        if self._fused(axis):
            return self._pattern.counts(self._rows, self._same)
        return super().sum(axis=axis, **kwargs)

    def any(self, axis=None, **kwargs):
        if self._fused(axis):
            return self._pattern.counts(self._rows, self._same) > 0
        return super().any(axis=axis, **kwargs)

    def mean(self, axis=None, **kwargs):
        if self._fused(axis):
            return self._pattern.counts(self._rows, self._same).to(torch.float64) / self._lens.to(torch.float64)
        return super().mean(axis=axis, **kwargs)


def _rolling(pattern: _Pattern, sequence, mode):
    if mode not in ("valid", "same"):
        raise ValueError(f"mode must be 'valid' or 'same', not {mode!r}")
    rows = pattern.rows(sequence)
    same = mode == "same"
    if rows.flat:
        return pattern.matches(rows, same)
    out = LazyMatches(pattern, rows, same)
    if not config.LAZY:
        out._data
    return out


def _windows(pattern: _Pattern, windows):
    """One bool per row of a 2-D array of windows as long as the pattern."""
    rows = pattern.rows(windows)
    if bool((rows.lens != pattern.span).any().item()):
        raise ValueError(f"windows must be {pattern.span} symbols long")
    out = pattern.matches(rows, False)
    return out[0] if rows.flat else out


class StringMatcher:
    """Matches of one literal string (string_matcher.py): every character is a symbol of ``encoding``."""

    def __init__(self, matching_sequence: str, encoding):
        self._pattern = _Pattern(matching_sequence, encoding, literal=True, gaps=False)
        self._encoding = encoding

    @property
    def window_size(self) -> int:
        return self._pattern.span

    def __call__(self, sequence):
        return _windows(self._pattern, sequence)

    def rolling_window(self, sequence, window_size: int = None, mode: str = "valid"):
        assert window_size in (None, self.window_size), "only the pattern's own windows"
        return _rolling(self._pattern, sequence, mode)


class FixedLenRegexMatcher(StringMatcher):
    """Matches of a pattern of literal symbols, ``.`` and ``[...]`` classes."""

    def __init__(self, matching_regex: str, encoding):
        self._pattern = _Pattern(matching_regex, encoding, gaps=False)
        self._encoding = encoding


class RegexMatcher(StringMatcher):
    """Matches of a pattern with gaps ``.{a,b}``: one value per position ("same" mode), True where some expansion
    matches and fits inside the row."""

    def __init__(self, matching_regex: str, encoding):
        self._pattern = _Pattern(matching_regex, encoding)
        self._encoding = encoding

    def rolling_window(self, sequence, window_size: int = None, mode: str = "same"):
        return _rolling(self._pattern, sequence, mode)


def match_string(sequence, matching_sequence: str):
    """Where ``matching_sequence`` occurs in the sequence(s): a bool RaggedArray with max(L - m + 1, 0) values per row
    of length L, or for a 1-D sequence a bool tensor of N - m + 1 values.  The pattern is encoded in the sequence's
    encoding: raw text compares bytes exactly; an AlphabetEncoding array takes letters of its alphabet, case-folded.

    >>> match_string(["ACGT", "TACTAC"], "AC").tolist()
    [[True, False, False], [False, True, False, False, True]]
    """
    if isinstance(sequence, (str, list, np.ndarray)):
        sequence = as_encoded_array(sequence)
    if not isinstance(sequence, (EncodedArray, EncodedRaggedArray)):
        raise TypeError(f"cannot match in {type(sequence)}")
    enc = sequence.encoding
    if not (enc.is_base_encoding() or isinstance(enc, AlphabetEncoding)):
        raise TypeError(f"match_string needs text or an AlphabetEncoding array, not {enc}")
    return StringMatcher(matching_sequence, enc).rolling_window(sequence)
