"""Records -> file text on the device (FastQBuffer.from_data / join_fields io/fastq_buffer.py:47-61,
OneLineBuffer.join_fields io/one_line_buffer.py:119-134, MultiLineFastaBuffer.from_data io/multiline_buffer.py:67-86)
and the writer ``bnp.open(path, "w")`` returns (NpBufferedWriter, io/parser.py:209-273).

The fields of the records stay where they are: each is a ragged view ``(base, starts, lens)`` -- names and qualities
usually into the raw chunk, sequences into the chunk or into a new tensor of codes -- plus an optional 256-byte table
applied on the way out (an AlphabetEncoding's codes -> letters, qualities v -> v + 33).  ``bnpk_format_offsets`` sizes
every entry and checks the sequence codes; ``bnpk_format_records`` writes any byte range of the text, so the writer
formats a large chunk in fixed-size slices, each copied into one of two pinned host buffers while a background thread
writes the previous one to the file."""
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import torch

from .. import _native as nv
from .. import ops
from ..encoded_array import BaseEncoding, EncodedArray, EncodedRaggedArray, as_encoded_array
from ..encodings.alphabet_encoding import AlphabetEncoding
from ..ragged import RaggedArray

SLICE_BYTES = 64 << 20          # output bytes formatted and copied to the host per step
_luts = {}


def _lut(kind, encoding, device):
    """256-entry device table: the letters of an alphabet's codes (0 for a byte that is not a code) or v -> v + 33."""
    key = (kind, repr(encoding), device.type, device.index)
    if key not in _luts:
        t = np.zeros(256, dtype=np.uint8)
        if kind == "alphabet":
            letters = np.array([ord(c) for c in encoding.get_alphabet()], dtype=np.uint8)
            t[:letters.size] = letters
        else:
            t = ((np.arange(256) + 33) & 255).astype(np.uint8)
        _luts[key] = torch.from_numpy(t).to(device)
    return _luts[key]


def _view(array):
    """(base uint8, starts int64, lens int32) of a ragged array (or a 1-D array as one row), no copy."""
    if isinstance(array, EncodedArray):
        data = array.raw().reshape(-1)
        return (data.contiguous(), torch.zeros(1, dtype=torch.int64, device=data.device),
                torch.full((1,), data.numel(), dtype=torch.int32, device=data.device))
    data = array._data.reshape(-1)
    if not data.is_cuda:
        raise nv.NativeLibraryError("writing needs CUDA tensors: bionumpy_b200 has no CPU fallback")
    if data.dtype != torch.uint8:
        if data.is_floating_point() or data.dtype == torch.bool:
            raise TypeError(f"cannot write values of dtype {data.dtype} as text")
        data = data.to(torch.uint8)
    return data.contiguous(), array._starts.contiguous(), array._lens.contiguous()


def _text_field(array, what):
    if isinstance(array, list):
        array = as_encoded_array(array)
    if not isinstance(array, (EncodedArray, EncodedRaggedArray)) or not array.encoding.is_base_encoding():
        raise TypeError(f"{what} must be text (BaseEncoding), got {getattr(array, 'encoding', type(array))}")
    return _view(array) + (None,)


def sequence_field(sequence):
    """Text is copied; the codes of an AlphabetEncoding are turned back into its letters."""
    if isinstance(sequence, list):
        sequence = as_encoded_array(sequence)
    if not isinstance(sequence, (EncodedArray, EncodedRaggedArray)):
        raise TypeError(f"a sequence must be an EncodedArray or EncodedRaggedArray, got {type(sequence).__name__}")
    enc = sequence.encoding
    if enc.is_base_encoding():
        return _view(sequence) + (None,)
    if not isinstance(enc, AlphabetEncoding):
        raise TypeError(f"cannot write a sequence in {enc}: only text and AlphabetEncoding codes are written")
    raw = sequence.raw() if isinstance(sequence, EncodedArray) else sequence._data
    if raw.dtype != torch.uint8 and raw.numel() and bool(((raw < 0) | (raw > 255)).any()):
        raise ValueError("sequence codes outside 0..255")
    base, starts, lens = _view(sequence)
    return base, starts, lens, _lut("alphabet", enc, base.device)


def quality_field(quality):
    """The FASTQ buffer's qualities (uint8, byte - 33); integers of another dtype must lie in 0..222."""
    if isinstance(quality, EncodedRaggedArray) and quality.encoding.is_base_encoding():
        return _view(quality) + (None,)
    if not isinstance(quality, RaggedArray) or isinstance(quality, EncodedRaggedArray):
        raise TypeError(f"a quality must be a RaggedArray of integers, got {type(quality).__name__}")
    data = quality._data
    if data.is_floating_point() or data.dtype == torch.bool:
        raise TypeError(f"qualities must be integers, got {data.dtype}")
    if data.dtype != torch.uint8 and data.numel():
        lo, hi = int(data.min().item()), int(data.max().item())
        if lo < 0 or hi > 222:
            raise ValueError(f"qualities must lie in 0..222 to be written as text, got {lo}..{hi}")
    base, starts, lens = _view(quality)
    return base, starts, lens, _lut("quality", None, base.device)


def entry_fields(entries, fmt):
    """The (name, sequence, quality) fields of a record chunk for format ``fmt``; FASTA drops the quality."""
    if not hasattr(entries, "name") or not hasattr(entries, "sequence"):
        raise TypeError(f"cannot write {type(entries).__name__}: it needs name and sequence fields")
    name = _text_field(entries.name, "a name")
    seq = sequence_field(entries.sequence)
    qual = None
    if fmt == nv.FMT_FASTQ:
        if not hasattr(entries, "quality"):
            raise ValueError("FASTQ needs a quality field: write SequenceEntry records as FASTA")
        qual = quality_field(entries.quality)
    counts = {f[2].numel() for f in (name, seq, qual) if f is not None}
    if len(counts) != 1:
        raise ValueError(f"the fields have different entry counts: {sorted(counts)}")
    return name, seq, qual


class Formatted:
    """The text of a record chunk: entry offsets on the device and its size; ``slice(a, b)`` formats bytes [a, b).
    A sequence code outside the alphabet raises EncodingError here, before any byte is formatted."""

    def __init__(self, fields, fmt, line_width):
        self.fields, self.fmt, self.line_width = fields, fmt, line_width
        self.offsets, status = ops.format_offsets(fmt, line_width, fields)
        self.size, st = ops.read_back(self.offsets[-1:], status)
        offset = st.bad_base_offset(fields[1][2])
        if offset is not None:
            from ..encodings import EncodingError
            raise EncodingError(f"Invalid sequence code at flat offset {offset}: it is not a letter of the alphabet",
                                offset)

    def slice(self, begin, end, out=None):
        return ops.format_records(self.fmt, self.line_width, self.fields, self.offsets, begin, end, out)


def formatted_entries(entries, fmt, line_width=1):
    """The text of a record chunk in a sequence format (the buffers' ``formatted``, which the writer calls)."""
    return Formatted(entry_fields(entries, fmt), fmt, line_width)


def format_entries(entries, fmt, line_width=1):
    """All of a chunk's text as one device tensor (the buffers' from_data)."""
    f = formatted_entries(entries, fmt, line_width)
    return EncodedArray(f.slice(0, f.size), BaseEncoding)


def join_fields(fields, fmt, line_width=1):
    """OneLineBuffer.join_fields: the text of name, sequence (and quality) arrays given as a list."""
    fields = list(fields)
    name = _text_field(fields[0], "a name")
    seq = sequence_field(fields[1])
    qual = None
    if fmt == nv.FMT_FASTQ:
        if len(fields) < 3:
            raise ValueError("FASTQ needs a quality field")
        q = fields[2]
        qual = _text_field(q, "a quality") if isinstance(q, EncodedRaggedArray) else quality_field(q)
    counts = {f[2].numel() for f in (name, seq, qual) if f is not None}
    if len(counts) != 1:
        raise ValueError(f"the fields have different entry counts: {sorted(counts)}")
    f = Formatted((name, seq, qual), fmt, line_width)
    return EncodedArray(f.slice(0, f.size), BaseEncoding)


class _HostSink:
    """Hands host byte slices to a file object in call order on one background thread; two pinned buffers are used in
    turn, so the device can fill one while the other is being written.  An error of the file is raised by the next
    call or by ``close``."""

    def __init__(self, file_obj):
        self._file = file_obj
        self._exec = ThreadPoolExecutor(1, thread_name_prefix="bnp-write")
        self._bufs = [None, None]
        self._pending = [None, None]
        self._turn = 0

    def _raise(self):
        for i, fut in enumerate(self._pending):
            if fut is not None and fut.done():
                self._pending[i] = None
                fut.result()

    def buffer(self, nbytes):
        """The next pinned buffer, once the write that used it last is done."""
        i = self._turn
        fut = self._pending[i]
        if fut is not None:
            self._pending[i] = None
            fut.result()
        self._raise()
        b = self._bufs[i]
        if b is None or b.numel() < nbytes:
            b = torch.empty(max(nbytes, 1 << 20), dtype=torch.uint8)
            if torch.cuda.is_available():
                b = b.pin_memory()
            self._bufs[i] = b
        return b

    def submit(self, buf, nbytes, event=None):
        """Write buf[:nbytes] after ``event`` (the copy into it) completes."""
        i = self._turn
        self._turn ^= 1

        def work():
            if event is not None:
                event.synchronize()
            self._file.write(memoryview(buf.numpy())[:nbytes])

        self._pending[i] = self._exec.submit(work)

    def flush(self):
        for i in (self._turn, self._turn ^ 1):
            fut = self._pending[i]
            if fut is not None:
                self._pending[i] = None
                fut.result()

    def close(self):
        try:
            self.flush()
        finally:
            self._exec.shutdown(wait=True)


class NpBufferedWriter:
    """parser.py:209-273: writes record chunks to a file object in the format of ``buffer_type``, whose
    ``formatted(chunk)`` gives the chunk's text: its ``size``, its line ``offsets`` on the device and
    ``slice(a, b, out)``, which formats bytes [a, b) into ``out``."""

    def __init__(self, file_obj, buffer_type):
        self._file_obj = file_obj
        self._buffer_type = buffer_type
        self._sink = _HostSink(file_obj)
        self._closed = False

    def __enter__(self):
        return self

    def __exit__(self, exc_type, exc_val, exc_tb):
        self.close()

    def close(self):
        if self._closed:
            return
        self._closed = True
        try:
            self._sink.close()
        finally:
            self._file_obj.close()

    def write(self, data):
        """A record chunk, a stream of them (``read_chunks()``, a generator) or a reader.  Returns once the bytes are on
        the host; the file receives them in call order."""
        from .parser import NpDataclassReader
        from ..streams import BnpStream
        import types
        if isinstance(data, NpDataclassReader):
            data = data.read_chunks()
        if isinstance(data, (BnpStream, types.GeneratorType)):
            for chunk in data:
                if len(chunk) > 0:
                    self.write(chunk)
            return
        if len(data) == 0:
            return
        f = self._buffer_type.formatted(data)
        dev = f.offsets.device
        with torch.cuda.device(dev):
            stream = torch.cuda.current_stream()
            step = max(int(SLICE_BYTES), 1)
            scratch = torch.empty(min(step, f.size), dtype=torch.uint8, device=dev)
            for a in range(0, f.size, step):
                b = min(f.size, a + step)
                host = self._sink.buffer(b - a)
                # the slice before this one was copied out of `scratch` on this stream: reuse is stream-ordered
                f.slice(a, b, scratch)
                host[:b - a].copy_(scratch[:b - a], non_blocking=True)
                ev = torch.cuda.Event()
                ev.record(stream)
                self._sink.submit(host, b - a, ev)
            stream.synchronize()
