"""BAM on the device (mirror of bionumpy/io/bam.py:18-366).

  header      : parsed on the host from the first inflated bytes (magic BAM\\1, l_text, the n_ref names and lengths);
                it may span several of the source's reads.  The names go to the device once, with "*" after them.
  split       : K15 bnpk_bam_split + bnpk_bam_fields on the chunk, then ONE synchronisation for the record count, the
                complete bytes and the first fault (FormatException naming the 0-based record of the file).
  get_data    : BamEntry fields built lazily from the kernel's outputs: text as (chunk, starts, lens) views, integers as
                int64, cigar ops / lengths and base codes unpacked by bnpk_bam_cigar / bnpk_bam_sequence, qualities as a
                view of the stored bytes.

Deviations from the reference: refID -1 gives the chromosome "*" (the reference indexes names[-1], the last contig);
BamIntervalBuffer leaves out records whose refID is -1; flag, position and mapq are int64."""
import struct

import torch

from .. import _native as nv
from .. import ops
from ..datatypes import BamEntry, Bed6
from ..encoded_array import EncodedArray, EncodedRaggedArray
from ..encodings import BamEncoding, CigarOpEncoding, StrandEncoding
from ..ragged import RaggedArray
from .buffers import FieldView
from .exceptions import FormatException

MAGIC = b"BAM\1"
FAULTS = {nv.BAM_BAD_BLOCK_SIZE: "block_size below 32",
          nv.BAM_BAD_REF_ID: "refID or next_refID outside the header's references",
          nv.BAM_BAD_NAME: "read name empty or not NUL-terminated",
          nv.BAM_BAD_SIZES: "the record's fields do not fit its block_size",
          nv.BAM_BAD_CIGAR_OP: "cigar op code above 8",
          nv.BAM_TRUNCATED: "the file ends inside a record"}


class BamHeader:
    """The header of a BAM file (BamHeader, io/bam.py:169-231): the SAM text, the reference names and lengths and the
    header's size in bytes.  ``info`` is the reference's list of (name, length)."""

    def __init__(self, text, names, lengths, size):
        self.text, self.names, self.lengths, self.size = text, names, lengths, size
        self.info = list(zip(names, lengths))
        self._device_names = {}

    def device_names(self, device):
        """(bytes, starts int64, lens int32) of the names and a last "*" on ``device``, copied once."""
        key = (device.type, device.index)
        if key not in self._device_names:
            names = [n.encode() for n in self.names] + [b"*"]
            lens = torch.tensor([len(n) for n in names], dtype=torch.int64)
            starts = torch.cumsum(lens, 0) - lens
            data = torch.frombuffer(bytearray(b"".join(names)), dtype=torch.uint8)
            self._device_names[key] = (data.to(device), starts.to(device), lens.to(torch.int32).to(device))
        return self._device_names[key]


def parse_header(data):
    """The BamHeader at the start of the inflated bytes ``data``, or None while they end inside it.  Raises
    FormatException when they do not start with BAM\\1 or a size in the header is negative."""
    n = len(data)
    if data[:min(n, 4)] != MAGIC[:min(n, 4)]:
        raise FormatException("not a BAM file: the inflated bytes do not start with BAM\\1", line_number=0)
    if n < 12:
        return None
    l_text = struct.unpack_from("<i", data, 4)[0]
    if l_text < 0:
        raise FormatException(f"BAM header: l_text {l_text} is negative", line_number=0)
    p = 8 + l_text
    if n < p + 4:
        return None
    text = bytes(data[8:p]).split(b"\0", 1)[0].decode("utf-8", "replace")
    n_ref = struct.unpack_from("<i", data, p)[0]
    if n_ref < 0:
        raise FormatException(f"BAM header: n_ref {n_ref} is negative", line_number=0)
    p += 4
    names, lengths = [], []
    for _ in range(n_ref):
        if n < p + 4:
            return None
        l_name = struct.unpack_from("<i", data, p)[0]
        if l_name < 1:
            raise FormatException(f"BAM header: reference name length {l_name}", line_number=0)
        if n < p + 8 + l_name:
            return None
        names.append(bytes(data[p + 4:p + 3 + l_name]).decode("utf-8", "replace"))
        lengths.append(struct.unpack_from("<i", data, p + 4 + l_name)[0])
        p += 8 + l_name
    return BamHeader(text, names, lengths, p)


def read_stream_header(source):
    """Reads a _Source (ingest.py) until its inflated bytes hold the whole header, doubling what it has read each time,
    so that at most the header's size of record bytes is read with it.  Returns (BamHeader, the bytes after the header,
    whether the source is exhausted)."""
    data = bytearray()
    while True:
        pinned, nread, last = source.finish(source.start(max(12, len(data))))
        data += memoryview(pinned.numpy())[:nread]
        header = parse_header(data)
        if header is not None:
            return header, bytes(data[header.size:]), last
        if last:
            raise FormatException("the file ends inside the BAM header", line_number=0)


class BamBuffer:
    """BamBuffer (io/bam.py:234-331): the complete records at the head of a chunk of inflated bytes on the device."""
    dataclass = BamEntry
    header = None               # the file's BamHeader, set by modify_class_with_header_data
    _final_newline = False      # binary records: the reader adds nothing to the last chunk

    def __init__(self, data, starts, fields, n_records, n_walked_again=0):
        self._data = data                   # device bytes, complete records only
        self._starts = starts               # int64[R] record offsets
        self._f = fields                    # int64[BAM_FIELDS, R] (bnpk_bam_fields)
        self._n = n_records
        self.n_walked_again = n_walked_again
        self._cache = {}

    # ---- protocol -----------------------------------------------------------------------------
    @classmethod
    def read_header(cls, file_object):
        """The header lies inside the compressed stream: the reader parses it (read_stream_header)."""
        return None

    @classmethod
    def modify_class_with_header_data(cls, header):
        if header is None:
            return cls
        return type(cls.__name__, (cls,), {"header": header})

    @classmethod
    def read_device_chunk(cls, d, last, n_before):
        """The complete records at the head of the device bytes ``d`` as a buffer, or None when ``d`` holds none.  A
        fault, and on the last chunk a record cut off by the end of the file, raises FormatException with the record's
        number in the file (``n_before`` records came before ``d``)."""
        if cls.header is None:
            raise ValueError("a BAM buffer needs the file's header: open the file with bnp.open")
        starts, status = ops.bam_split(d, len(cls.header.names))
        fields = ops.bam_fields(d, starts, status)
        st = ops.read_status(status)                                 # the one synchronisation of this chunk
        n, size, fault = st.n_records, st.n_complete_bytes, st.words[nv.ST_BAD_BASE]
        if fault == nv.INT64_MAX and last and size < d.numel():
            fault = n << 8 | nv.BAM_TRUNCATED
        if fault != nv.INT64_MAX:
            record = n_before + (fault >> 8)
            raise FormatException(f"BAM record {record}: {FAULTS.get(fault & 255, 'invalid record')}",
                                  line_number=record)
        if n == 0:
            return None
        return cls(d[:size], starts[:n], fields[:, :n], n, st.n_values)

    @classmethod
    def concatenate(cls, buffers):
        """One buffer of the records of consecutive chunks."""
        data = torch.cat([b._data for b in buffers])
        shift, starts, fields = 0, [], []
        moved = torch.tensor([f in (nv.BAM_F_NAME_START, nv.BAM_F_CIGAR_START, nv.BAM_F_SEQ_START, nv.BAM_F_QUAL_START)
                              for f in range(nv.BAM_FIELDS)], device=data.device).to(torch.int64)[:, None]
        for b in buffers:
            starts.append(b._starts + shift)
            fields.append(b._f + moved * shift)
            shift += b._data.numel()
        return cls(data, torch.cat(starts), torch.cat(fields, 1), sum(b._n for b in buffers),
                   sum(b.n_walked_again for b in buffers))

    @property
    def size(self) -> int:
        return self._data.numel()

    @property
    def n_lines(self) -> int:
        return self._n

    def count_entries(self) -> int:
        return self._n

    def __len__(self):
        return self._n

    def get_data(self):
        return self.dataclass.lazy(self)

    # ---- fields (BamBufferExtractor, io/bam.py:18-166) --------------------------------------------
    def _row(self, f):
        return self._f[f]

    def _chromosome(self):
        data, starts, lens = self.header.device_names(self._data.device)
        ref = self._row(nv.BAM_F_REF_ID)
        ids = torch.where(ref < 0, len(self.header.names), ref)          # refID -1: the "*" after the names
        return FieldView(data, lens[ids], starts[ids])

    def _cigar(self):
        if "cigar" not in self._cache:
            n_cigar = self._row(nv.BAM_F_N_CIGAR)
            offsets = ops.row_offsets(n_cigar.to(torch.int32))
            op, length = ops.bam_cigar(self._data, self._row(nv.BAM_F_CIGAR_START), offsets, int(offsets[-1].item()))
            self._cache["cigar"] = (EncodedRaggedArray(EncodedArray(op, CigarOpEncoding), n_cigar),
                                    RaggedArray(length, n_cigar))
        return self._cache["cigar"]

    def _sequence(self):
        l_seq = self._row(nv.BAM_F_L_SEQ)
        offsets = ops.row_offsets(l_seq.to(torch.int32))
        codes = ops.bam_sequence(self._data, self._row(nv.BAM_F_SEQ_START), offsets, int(offsets[-1].item()))
        return EncodedRaggedArray(EncodedArray(codes, BamEncoding), l_seq)

    def get_field_by_number(self, i, t=None):
        if i not in self._cache:
            if i == 0:
                v = self._chromosome()
            elif i == 1:
                v = FieldView(self._data, self._row(nv.BAM_F_NAME_LEN), self._row(nv.BAM_F_NAME_START))
            elif i in (2, 3, 4):
                v = self._row((nv.BAM_F_FLAG, nv.BAM_F_POS, nv.BAM_F_MAPQ)[i - 2])
            elif i in (5, 6):
                v = self._cigar()[i - 5]
            elif i == 7:
                v = self._sequence()
            elif i == 8:
                v = RaggedArray(self._data, self._row(nv.BAM_F_L_SEQ), starts=self._row(nv.BAM_F_QUAL_START))
            else:
                raise IndexError(i)
            self._cache[i] = v
        return self._cache[i]


class BamIntervalBuffer(BamBuffer):
    """BamIntervalBuffer (io/bam.py:334-366): every placed alignment as a Bed6 row: chromosome, start = pos,
    stop = pos + the reference length of its cigar (summed on the device, so the cigar arrays are never built), name,
    score = mapq, strand '-' where flag 0x10 is set.  Records whose refID is -1 have no place on the reference and are
    left out; placed unmapped reads keep their zero-length interval, as in the reference."""
    dataclass = Bed6

    def _placed(self):
        if "placed" not in self._cache:
            self._cache["placed"] = torch.nonzero(self._f[nv.BAM_F_REF_ID] >= 0).squeeze(1)
        return self._cache["placed"]

    def count_entries(self) -> int:
        return self._placed().numel()

    def __len__(self):
        return self.count_entries()

    def _row(self, f):
        return self._f[f][self._placed()]

    def get_field_by_number(self, i, t=None):
        if i not in self._cache:
            if i == 0:
                v = self._chromosome()
            elif i == 3:
                v = FieldView(self._data, self._row(nv.BAM_F_NAME_LEN), self._row(nv.BAM_F_NAME_START))
            elif i == 1:
                v = self._row(nv.BAM_F_POS)
            elif i == 2:
                v = self._row(nv.BAM_F_POS) + self._row(nv.BAM_F_REF_LEN)
            elif i == 4:
                v = self._row(nv.BAM_F_MAPQ)
            elif i == 5:
                v = EncodedArray(((self._row(nv.BAM_F_FLAG) & 16) != 0).to(torch.uint8), StrandEncoding)
            else:
                raise IndexError(i)
            self._cache[i] = v
        return self._cache[i]
