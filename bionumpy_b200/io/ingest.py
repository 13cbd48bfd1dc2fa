"""Host -> device ingest for the chunk reader (SURVEY 8f-1; replaces, for plain and gzip-compressed FASTQ / FASTA
files, NumpyFileReader.read_chunk's np.concatenate + the pageable cp.asanyarray of the cupy reader:
bionumpy/io/parser.py:96-171, bionumpy/cupy_compatible/parser.py:10-17, bionumpy/io/gzip_reading.py:1-4).

  PinnedFileReader   plain files: the next chunk is pread() by a pool of threads straight into a pinned staging
                     buffer WHILE the GPU works on the current one; one async H2D per chunk; the tail that belongs to
                     the next chunk never leaves the device (no host concatenation); the line census that finds the
                     last complete entry is the only synchronisation per chunk and its result builds the buffer
                     (from_raw_buffer's own census is skipped).
  inflate_stream     .gz input: BGZF (bgzip) files are inflated block-parallel on the host cores (zlib releases the
                     GIL) in file order; ordinary single-member gzip is inflated by one background thread.  Either
                     way inflation overlaps the GPU's work on the previous chunk and fills pinned buffers.
Same chunking semantics as the reference reader: chunks hold complete entries only, at least min_chunk_size bytes are
read per chunk, the tail is carried over, the last chunk gets its '\\n'.
"""
import os
import struct
import threading
import zlib
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import torch

from .. import config, ops
from .exceptions import FormatException
from .parser import CudaFileReader

NEWLINE = 10
_POOL = None


def _pool():
    global _POOL
    if _POOL is None:
        n = int(os.environ.get("BNP_INGEST_THREADS", "0")) or \
            max(4, min(48, len(os.sched_getaffinity(0)) if hasattr(os, "sched_getaffinity") else (os.cpu_count() or 4)))
        _POOL = ThreadPoolExecutor(n, thread_name_prefix="bnp-ingest")
    return _POOL


class _Staging:
    """Two pinned host buffers used in turn (one being filled by the readers, one being copied to the device)."""

    def __init__(self):
        self._bufs = [None, None]
        self._turn = 0

    def take(self, nbytes):
        i = self._turn
        self._turn ^= 1
        b = self._bufs[i]
        if b is None or b.numel() < nbytes:
            b = torch.empty(max(nbytes, 1 << 20), dtype=torch.uint8)
            if torch.cuda.is_available():
                b = b.pin_memory()
            self._bufs[i] = b
        return b


class _Source:
    """start(nbytes) begins filling a pinned buffer with the next `nbytes` (or fewer at the end) of the byte stream and
    returns a handle; finish(handle) -> (pinned tensor, bytes filled, stream exhausted)."""

    def close(self):
        pass


class _PreadSource(_Source):
    def __init__(self, file_obj):
        self._file = file_obj                          # keeps the descriptor open
        self._fd = file_obj.fileno()
        self._pos = file_obj.tell()
        self._size = os.fstat(self._fd).st_size
        self._staging = _Staging()

    def start(self, nbytes):
        nbytes = max(0, min(nbytes, self._size - self._pos))
        buf = self._staging.take(nbytes)
        mv = memoryview(buf.numpy())
        piece = max(1 << 20, min(8 << 20, -(-nbytes // 32)))
        futs = []
        for a in range(0, nbytes, piece):
            b = min(nbytes, a + piece)
            futs.append(_pool().submit(self._read_piece, mv[a:b], self._pos + a))
        self._pos += nbytes
        return buf, nbytes, futs, self._pos >= self._size

    def _read_piece(self, view, offset):
        done = 0
        while done < len(view):
            got = os.preadv(self._fd, [view[done:]], offset + done)
            if got <= 0:
                raise IOError("short read")
            done += got

    def finish(self, handle):
        buf, nbytes, futs, last = handle
        for f in futs:
            f.result()
        return buf, nbytes, last


def _bgzf_blocks(raw: memoryview):
    """[(payload offset, payload size, uncompressed size)] of a BGZF file image, or None if it is not BGZF (every member
    must carry the 'BC' extra field, SAM spec 4.1)."""
    blocks, p, n = [], 0, len(raw)
    while p < n:
        if n - p < 18 or raw[p] != 0x1F or raw[p + 1] != 0x8B or raw[p + 2] != 8 or not (raw[p + 3] & 4):
            return None
        xlen = struct.unpack_from("<H", raw, p + 10)[0]
        q, end, bsize = p + 12, p + 12 + xlen, None
        while q + 4 <= end:
            si1, si2, slen = raw[q], raw[q + 1], struct.unpack_from("<H", raw, q + 2)[0]
            if si1 == 66 and si2 == 67 and slen == 2:
                bsize = struct.unpack_from("<H", raw, q + 4)[0] + 1
            q += 4 + slen
        if bsize is None or p + bsize > n:
            return None
        isize = struct.unpack_from("<I", raw, p + bsize - 4)[0]
        blocks.append((p + 12 + xlen, bsize - xlen - 20, isize))
        p += bsize
    return blocks


class _GzipSource(_Source):
    """Inflates a .gz file ahead of the consumer into pinned buffers: block-parallel for BGZF, one background thread for
    ordinary gzip (a single DEFLATE stream cannot be split)."""

    def __init__(self, path):
        self._staging = _Staging()
        with open(path, "rb") as f:
            self._raw = f.read()                       # compressed bytes: ~1/4 of the text
        self._blocks = _bgzf_blocks(memoryview(self._raw))
        self.parallel = self._blocks is not None
        self._next_block = 0
        self._excess = b""                             # inflated bytes beyond the requested count (BGZF: whole blocks)
        self._carry = b""
        self._z = None if self.parallel else zlib.decompressobj(wbits=31)
        self._zpos = 0
        self._eof = False

    # -- BGZF: whole blocks, inflated in parallel straight into the pinned buffer --------------------------------
    def _inflate_block(self, view, off, size):
        out = zlib.decompress(self._raw[off:off + size], wbits=-15)
        view[:len(out)] = out

    def start(self, nbytes):
        if self.parallel:
            take, total = [], len(self._excess)
            while self._next_block < len(self._blocks) and total < nbytes:
                b = self._blocks[self._next_block]
                take.append((total,) + b)
                total += b[2]
                self._next_block += 1
            buf = self._staging.take(total)
            mv = memoryview(buf.numpy())
            mv[:len(self._excess)] = self._excess
            self._excess = b""
            futs = [_pool().submit(self._inflate_block, mv[o:o + isz], off, size) for o, off, size, isz in take if isz]
            return buf, (total, nbytes), futs, self._next_block >= len(self._blocks)
        # single stream: one worker inflates the next nbytes while the caller does something else
        buf = self._staging.take(nbytes + (1 << 16))
        fut = _pool().submit(self._inflate_stream, buf, nbytes)
        return buf, None, [fut], None

    def _inflate_stream(self, buf, nbytes):
        mv = memoryview(buf.numpy())
        filled = 0
        if self._carry:
            k = min(len(self._carry), len(mv))
            mv[:k] = self._carry[:k]
            self._carry = self._carry[k:]
            filled = k
        raw = self._raw
        while filled < nbytes and not self._eof:
            if self._z.eof:                            # multi-member gzip: the next member starts here
                rest = self._z.unused_data
                if not rest:
                    self._eof = True
                    break
                self._z = zlib.decompressobj(wbits=31)
                out = self._z.decompress(rest, nbytes - filled)
            else:
                piece = b"" if self._z.unconsumed_tail else raw[self._zpos:self._zpos + (1 << 20)]
                self._zpos += len(piece)
                if not piece and not self._z.unconsumed_tail:
                    self._eof = True
                    break
                out = self._z.decompress(self._z.unconsumed_tail + piece, nbytes - filled)
            mv[filled:filled + len(out)] = out
            filled += len(out)
        return filled, self._eof and not self._carry

    def finish(self, handle):
        buf, total, futs, last = handle
        if self.parallel:
            for f in futs:
                f.result()
            have, want = total
            if have > want:                            # hand out exactly what was asked for, like file.read(n)
                self._excess = bytes(memoryview(buf.numpy())[want:have])
                return buf, want, False
            return buf, have, last
        filled, eof = futs[0].result()
        return buf, filled, eof


class PinnedFileReader(CudaFileReader):
    """The chunk reader over a _Source (plain file or inflated gzip) for the one-line buffer types and BAM.  The buffer
    type finds the complete entries of each chunk (``read_device_chunk``) and joins chunks (``concatenate``)."""

    def __init__(self, file_obj, buffer_type, source):
        super().__init__(file_obj, buffer_type)
        self._source = source
        self._pending = None
        self._tail = None                              # device bytes that belong to the next chunk
        self._tail_last = NEWLINE                      # the tail's last byte, known on the host
        self._exhausted = False                        # the header read the whole stream
        if hasattr(buffer_type, "header"):             # BAM: the header lies inside the inflated stream
            from .bam import read_stream_header
            self._header_data, rest, self._exhausted = read_stream_header(source)
            self._buffer_type = buffer_type.modify_class_with_header_data(self._header_data)
            if rest:
                self._tail = torch.frombuffer(bytearray(rest), dtype=torch.uint8).to(config.default_device())

    def close(self):
        self._source.close()
        super().close()

    def read(self):
        chunks = []
        while True:
            b = self.read_chunk(min_chunk_size=64 << 20)
            if b is None:
                break
            chunks.append(b)
        if not chunks:
            return None
        if len(chunks) == 1:
            return chunks[0]
        return self._buffer_type.concatenate(chunks)

    def read_chunk(self, min_chunk_size: int = 5000000, max_chunk_size: int = None):
        if self._is_finished:
            return None
        bt = self._buffer_type
        dev = config.default_device()
        while True:
            if self._exhausted:
                pinned, nread, last = None, 0, True
            else:
                handle = self._pending if self._pending is not None else self._source.start(min_chunk_size)
                self._pending = None
                pinned, nread, last = self._source.finish(handle)
                if not last:
                    self._pending = self._source.start(min_chunk_size)  # the next chunk fills while the GPU works
            tail_len = 0 if self._tail is None else self._tail.numel()
            total = tail_len + nread
            if total == 0:
                self._is_finished = True
                return None
            last_byte = int(pinned[nread - 1]) if nread else self._tail_last
            add_nl = last and last_byte != NEWLINE and bt._final_newline   # parser.py:183-186
            d = torch.empty(total + (1 if add_nl else 0), dtype=torch.uint8, device=dev)
            if tail_len:
                d[:tail_len] = self._tail
            if nread:
                d[tail_len:total].copy_(pinned[:nread], non_blocking=True)
            if add_nl:
                d[total:] = NEWLINE
                last_byte = NEWLINE
            if max_chunk_size is not None and d.numel() > max_chunk_size:
                raise Exception("No complete entry found")
            buff = bt.read_device_chunk(d, last, self.n_lines_read)      # the one synchronisation of this chunk
            if buff is None:
                if last:
                    self._is_finished = True
                    return None
                self._tail, self._tail_last = d, last_byte               # no complete entry yet: read more
                continue
            size = buff.size
            self._tail = None if last or size == d.numel() else d[size:].clone()
            self._tail_last = last_byte
            self._is_finished = last
            self.n_bytes_read += size
            self.n_lines_read += buff.n_lines
            return buff


def open_reader(path, file_obj, buffer_type, is_gzip):
    """The ingest reader for `path` if the buffer type is one of the one-line CUDA buffers or BAM, else None.  BAM is
    always read as BGZF (or gzip)."""
    from .bam import BamBuffer
    from .buffers import CudaOneLineBuffer
    if isinstance(buffer_type, type) and issubclass(buffer_type, BamBuffer):
        if file_obj.read(2) != b"\x1f\x8b":
            file_obj.close()
            raise FormatException(f"{path} is not a BAM file: BAM is BGZF-compressed, and this file is not gzip")
        file_obj.seek(0)
        return PinnedFileReader(file_obj, buffer_type, _GzipSource(path))
    if not (isinstance(buffer_type, type) and issubclass(buffer_type, CudaOneLineBuffer)):
        return None
    if is_gzip:
        return PinnedFileReader(file_obj, buffer_type, _GzipSource(path))
    try:
        file_obj.fileno()
    except Exception:
        return None
    return PinnedFileReader(file_obj, buffer_type, _PreadSource(file_obj))
