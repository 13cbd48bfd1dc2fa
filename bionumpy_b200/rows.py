"""The ragged byte view the row-driven kernels read (csrc/row_kernels.cu): rows ``(base, starts, lens)`` of one uint8
CUDA tensor, how the kernels read them (``enc_mode``, ``lut``), and the alphabet a bad base is reported in.  K-mers,
minimizers, exact counts, motif scores, encoding and reverse complement all build their kernel input here."""
import copy

import torch

from . import _native as nv
from . import ops
from .encoded_array import EncodedArray

LONG_ROW = 1 << 14          # rows longer than this are cut into overlapping pieces, one warp each


def _long_row_pieces(starts, lens, span, out_offsets=None, piece=LONG_ROW):
    """Rows longer than ``piece`` positions become pieces [i*piece, (i+1)*piece + span - 1): every k-mer /
    window start belongs to exactly one piece, so counts and (with ``out_offsets``) materialised values are
    unchanged while long rows (chromosomes) spread over many warps.  Index arithmetic only (torch);
    returns (starts, lens, out_offsets, row) of the pieces, ``row`` the row each piece comes from (None: no split)."""
    L = lens.to(torch.int64)
    if L.numel() == 0 or int(L.max().item()) <= piece + span - 1:
        return starts, lens, out_offsets, None
    n_pos = torch.clamp(L - (span - 1), min=0)                       # window starts per row
    n_pieces = torch.clamp((n_pos + piece - 1) // piece, min=1)
    row = torch.repeat_interleave(torch.arange(L.numel(), device=L.device), n_pieces)
    first = torch.cumsum(n_pieces, 0) - n_pieces
    idx = torch.arange(row.numel(), device=L.device) - first[row]    # piece index inside its row
    p_start = starts[row] + idx * piece
    p_len = torch.minimum(L[row] - idx * piece, torch.full_like(idx, piece + span - 1))
    p_off = None if out_offsets is None else out_offsets[:-1][row] + idx * piece
    return p_start.contiguous(), p_len.to(torch.int32).contiguous(), p_off, row


def _split_long_rows(starts, lens, span, out_offsets=None, piece=LONG_ROW):
    """(starts, lens, out_offsets) of the pieces of ``_long_row_pieces``, for callers that launch on the pieces alone."""
    return _long_row_pieces(starts, lens, span, out_offsets, piece)[:3]


class RowView:
    """Rows of ``base`` (contiguous uint8 CUDA) at ``starts`` (int64) with ``lens`` (int32 bases).

    ``RowView(sequence, text_encoding)``: a 1-D EncodedArray is one row (``flat``), a 2-D one has a row per line, an
    EncodedRaggedArray keeps its own view.  Text (BaseEncoding) is read into ``text_encoding``; an array that is
    already encoded is read as its codes (ENC_CODES).  ``alphabet_encoding`` is the alphabet of the codes the kernels
    see: a bad base is reported in it.  ``chunk_buffer`` is the file buffer when the view is an untouched field of one."""

    def __init__(self, sequence, text_encoding=None):
        if isinstance(sequence, EncodedArray):
            data = sequence.raw()
            if data.dim() == 1:
                starts = torch.zeros(1, dtype=torch.int64, device=data.device)
                lens = torch.full((1,), data.numel(), dtype=torch.int32, device=data.device)
            else:
                n, w = data.shape
                starts = torch.arange(n, dtype=torch.int64, device=data.device) * w
                lens = torch.full((n,), w, dtype=torch.int32, device=data.device)
            data, self.flat = data.reshape(-1).contiguous(), data.dim() == 1
        else:
            data, starts, lens = sequence._data.contiguous(), sequence._starts.contiguous(), sequence._lens.contiguous()
            self.flat = False
        if not data.is_cuda:
            raise nv.NativeLibraryError("the row kernels need CUDA tensors: bionumpy_b200 has no CPU fallback")
        if data.dtype != torch.uint8:
            data = data.to(torch.uint8)
        self.base, self.starts, self.lens = data, starts, lens
        if sequence.encoding.is_base_encoding():
            self.alphabet_encoding = text_encoding
            self.enc_mode = None if text_encoding is None else text_encoding.enc_mode
            self.lut = text_encoding.device_lut(data.device) if self.enc_mode == nv.ENC_LUT else None
        else:
            self.alphabet_encoding, self.enc_mode, self.lut = sequence.encoding, nv.ENC_CODES, None
        self.chunk_buffer = getattr(sequence, "_chunk_buffer", None)

    def split(self, span, offsets=None):
        """Long rows cut into pieces of LONG_ROW window starts (``span`` bases per window), each a row of the returned
        view.  Returns ``(pieces, offsets, total, piece_row)``: ``offsets`` are the rows' output offsets (exclusive
        prefix sums of their windows, int64[R+1]) turned into the pieces' (int64[P+1]: the kernels read
        ``offsets[piece]`` only), ``total`` their last entry and ``piece_row`` the row of each piece.  When no row is
        long, this view, ``offsets``, None and None."""
        starts, lens, p_off, row = _long_row_pieces(self.starts, self.lens, span, offsets)
        if row is None:
            return self, offsets, None, None
        total = None
        if offsets is not None:
            total = int(offsets[-1].item())
            p_off = torch.cat([p_off, offsets[-1:]]).contiguous()
        pieces = copy.copy(self)
        pieces.starts, pieces.lens, pieces.chunk_buffer = starts, lens, None
        return pieces, p_off, total, row

    def raise_bad_base(self, status, rescan=None):
        """Raise the reference's EncodingError(offset) if ``status`` (a device status block, or a ScanStatus already
        read) reports a byte outside the alphabet.  When the launch ran on other rows than these (pieces, batches),
        ``rescan(view) -> status`` finds the (row, position) again on these rows first (error path).  A row past the
        last one, which a fused chunk count can report, is not a bad base of these rows."""
        if not isinstance(status, ops.ScanStatus):
            status = ops.read_status(status)
        if rescan is not None and status.bad_base() is not None:
            status = ops.read_status(rescan(self))
        bad = status.bad_base(self.lens.numel())
        if bad is not None:
            self.alphabet_encoding._raise_encoding_error(bad[0], bad[1], self.lens)
