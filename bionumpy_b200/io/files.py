"""bnp.open for the sequence formats of the hot path (mirror of bionumpy/io/files.py:28-227):
suffix -> buffer type, ``.gz`` detection, reader or writer construction, count_entries.  ``buffer_type=`` injects any
class honouring the FileBuffer protocol, exactly as in the reference (files.py:52-68)."""
import gzip
import os

from .buffers import CudaFastQBuffer, CudaTwoLineFastaBuffer
from .parser import CudaFileReader, NpDataclassReader

buffer_types = {
    ".fq": CudaFastQBuffer,
    ".fastq": CudaFastQBuffer,
}

WRITE_MODES = {"w": "wb", "wb": "wb", "write": "wb", "a": "ab", "ab": "ab", "append": "ab"}


def _multiline():
    from .multiline import CudaMultiLineFastaBuffer
    return CudaMultiLineFastaBuffer


def _buffer_type_for(suffix):
    if suffix in buffer_types:
        return buffer_types[suffix]
    if suffix in (".fa", ".fasta", ".fna", ".faa"):
        return _multiline()
    if suffix == ".bed":
        from .delimited import BedBuffer
        return BedBuffer
    if suffix == ".bdg":
        from .delimited import BdgBuffer
        return BdgBuffer
    if suffix == ".bam":
        from .bam import BamBuffer
        return BamBuffer
    raise RuntimeError(f"File format {suffix} does not have a default buffer type on the CUDA path "
                       f"(supported: .fq .fastq .fa .fasta .bed .bdg and their .gz forms, and .bam); pass buffer_type=")


def _suffix(path):
    base, suffix = os.path.splitext(path)
    is_gzip = suffix == ".gz"
    if is_gzip:
        suffix = os.path.splitext(base)[1]
    return suffix, is_gzip


def bnp_open(filename, mode=None, buffer_type=None, lazy=None):
    """files.py:85-182.  Reading ("r", "rb") gives an NpDataclassReader; writing ("w", "wb", "write") or appending
    ("a", "ab", "append") gives an NpBufferedWriter, which writes ``.gz`` files as BGZF.  ``.bdg`` (bedGraph) is
    written only, ``.bam`` read only (as BGZF, whatever the suffix says).  BED is written with the buffer type named: ``bnp.open("x.bed", "w", buffer_type=BedBuffer)`` (or
    Bed6Buffer; either writes a record's own fields).  Opening ``.bed`` for writing by its suffix alone raises
    NotImplementedError, as it did before BED could be written, so code that relies on that keeps working."""
    if mode not in (None, "r", "rb") and mode not in WRITE_MODES:
        raise NotImplementedError(f"mode {mode!r}: use r/rb to read, w/wb/write or a/ab/append to write")
    path = str(filename)
    suffix, is_gzip = _suffix(path)
    if mode in WRITE_MODES and buffer_type is None and suffix == ".bam":      # BAM is read only
        raise RuntimeError(f"File format {suffix} does not have a default buffer type on the CUDA path "
                           f"(supported: .fq .fastq .fa .fasta .bed .bdg and their .gz forms); pass buffer_type=")
    if mode in WRITE_MODES and buffer_type is None and suffix == ".bed":
        raise NotImplementedError("writing .bed by its suffix alone is not supported: name the format with "
                                  "buffer_type=bnp.io.BedBuffer (or Bed6Buffer)")
    if buffer_type is None:
        buffer_type = _buffer_type_for(suffix)
    if mode in WRITE_MODES:
        from .write import NpBufferedWriter
        raw = open(path, WRITE_MODES[mode])
        if is_gzip:
            from .bgzf import BgzfWriter
            raw = BgzfWriter(raw)
        return NpBufferedWriter(raw, buffer_type)
    from . import ingest
    raw = open(path, "rb")
    reader = ingest.open_reader(path, raw, buffer_type, is_gzip)        # pinned, prefetching ingest (FASTQ / 2-line FASTA)
    if reader is None:
        if is_gzip:
            raw.close()
            raw = gzip.open(path, "rb")
        reader = CudaFileReader(raw, buffer_type)
    return NpDataclassReader(reader, lazy)


def count_entries(filename, buffer_type=None) -> int:
    """files.py:185-227: the number of entries in the file, the sum of its chunks' count_entries()."""
    with bnp_open(filename, buffer_type=buffer_type) as f:
        return sum(buff.count_entries() for buff in f._reader.read_chunks(min_chunk_size=5000000))
