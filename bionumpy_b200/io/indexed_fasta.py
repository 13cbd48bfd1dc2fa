"""IndexedFasta on the device (mirror of bionumpy/io/indexed_fasta.py:13-206).

The FASTA file is brought to the device once (pinned, prefetching ingest); a set of intervals is then one gather that
checks every interval against its contig and skips the line ends (bnpk_interval_gather, through ops.interval_gather),
and a whole contig is the consecutive intervals that cover it -- where the reference seeks and reads per interval and
deletes the newline bytes on the host (indexed_fasta.py:101-131, 133-206).  The index is the .fai next to the file
(read_index, indexed_fasta.py:13-31); without one it is built from the file image (create_index, :34-58: name, length,
offset of the first base, bases per line, bytes per line)."""
import os
from pathlib import Path

import numpy as np
import torch

from .. import _native as nv
from .. import config, ops
from ..encoded_array import EncodedArray, EncodedRaggedArray, BaseEncoding
from ..rows import RowView

# Bases per interval of a whole-contig fetch.  The gather gives a row eight lanes, so a contig goes as many short rows:
# the 1.53 Mbases of sacCer3's chrIV take 36 ms as one row and 0.24-0.37 ms as rows of 1024 (as of 256; 0.68 ms as rows
# of 16384) on an H100 80GB HBM3 at a 700 W power limit.
_PIECE = 1024


def read_index(filename) -> dict:
    """indexed_fasta.py:13-31."""
    out = {}
    for line in open(filename):
        chromosome, rlen, offset, lenc, lenb = line.rstrip("\n").split("\t")[:5]
        out[chromosome.split()[0]] = {"rlen": int(rlen), "offset": int(offset), "lenc": int(lenc), "lenb": int(lenb)}
    return out


def create_index(filename) -> dict:
    """indexed_fasta.py:34-58 as a dict like read_index: one pass over the host bytes (index building is not on the
    hot path; the reference streams FastaIdxBuffer chunks)."""
    data = np.fromfile(str(filename), dtype=np.uint8)
    nl = np.flatnonzero(data == 10)
    line_starts = np.insert(nl[:-1] + 1, 0, 0) if nl.size else np.zeros(1, dtype=np.int64)
    if nl.size == 0 or nl[-1] != data.size - 1:
        line_starts = np.append(line_starts, nl[-1] + 1) if nl.size else line_starts
        nl = np.append(nl, data.size)
    is_hdr = data[line_starts] == ord(">")
    hdr_idx = np.flatnonzero(is_hdr)
    out = {}
    for n, h in enumerate(hdr_idx):
        end = hdr_idx[n + 1] if n + 1 < hdr_idx.size else line_starts.size
        name = bytes(data[line_starts[h] + 1:nl[h]]).decode().split()[0] if nl[h] > line_starts[h] + 1 else ""
        if end == h + 1:
            out[name] = {"rlen": 0, "offset": int(nl[h] + 1), "lenc": 0, "lenb": 0}
            continue
        first = h + 1
        line_len = nl[first:end] - line_starts[first:end]
        cr = (data[np.maximum(nl[first:end] - 1, 0)] == 13) & (line_len > 0)
        lenc = int(line_len[0] - cr[0])
        lenb = int(nl[first] + 1 - line_starts[first])
        out[name] = {"rlen": int((line_len - cr).sum()), "offset": int(line_starts[first]), "lenc": lenc, "lenb": lenb}
    return out


class IndexedFasta:
    """Behaves like a dict of chromosome names to sequences (indexed_fasta.py:61-131)."""

    def __init__(self, filename):
        filename = Path(filename)
        self._filename = filename
        fai = filename.with_suffix(filename.suffix + ".fai")
        self._index = read_index(fai) if fai.exists() else create_index(filename)
        dev = config.default_device()
        if dev.type != "cuda":
            raise nv.NativeLibraryError("IndexedFasta needs a CUDA device: bionumpy_b200 has no CPU fallback")
        from . import ingest
        with open(filename, "rb") as f:
            src = ingest._PreadSource(f)
            pinned, n, _ = src.finish(src.start(os.path.getsize(filename)))
            self._file = pinned[:n].to(dev, non_blocking=True)
            torch.cuda.current_stream().synchronize()

    def get_contig_lengths(self):
        return {name: values["rlen"] for name, values in self._index.items()}

    def keys(self):
        return self._index.keys()

    def values(self):
        return (self[key] for key in self.keys())

    def items(self):
        return ((key, self[key]) for key in self.keys())

    def __repr__(self):
        return f"Indexed Fasta File with chromosome sizes: {self.get_contig_lengths()}"

    def __getitem__(self, chromosome: str) -> EncodedArray:
        """The whole sequence of a contig (indexed_fasta.py:101-131): its consecutive intervals of _PIECE bases, whose
        rows lie one after the other in the gather's output."""
        rlen = self._index[chromosome]["rlen"]
        contig_ids, _, _, contigs = self._name_table()
        start = torch.arange(0, rlen, _PIECE, dtype=torch.int64, device=self._file.device)
        stop = (start + _PIECE).clamp(max=rlen)
        ids = torch.full_like(start, contig_ids[chromosome], dtype=torch.int32)
        out, _, bad, _ = ops.interval_gather(self._file, start, stop, ids, contigs)
        if bad is not None:
            raise AssertionError(f"contig {chromosome} reaches beyond the file")
        return EncodedArray(out, BaseEncoding)

    def _name_table(self):
        """The contig names sorted as bytes: each name's place in that order (the contig id), the names concatenated
        on the device with their offsets, and each contig's (offset, lenc, lenb, length) by id: built once, for
        bnpk_name_lookup and bnpk_interval_gather."""
        if getattr(self, "_table", None) is None:
            dev = self._file.device
            names = sorted(self._index, key=lambda n: n.encode())
            raw = [n.encode() for n in names]
            ends = np.cumsum([0] + [len(b) for b in raw]).astype(np.int64)
            idx = [self._index[n] for n in names]
            t = lambda v, dt: torch.tensor(v, dtype=dt, device=dev)
            text = torch.frombuffer(bytearray(b"".join(raw) or b"\0"), dtype=torch.uint8).to(dev)
            contigs = (t([i["offset"] for i in idx], torch.int64), t([i["lenc"] for i in idx], torch.int32),
                       t([i["lenb"] for i in idx], torch.int32), t([i["rlen"] for i in idx], torch.int64))
            self._table = ({n: k for k, n in enumerate(names)}, text, torch.from_numpy(ends).to(dev), contigs)
        return self._table

    def get_interval_sequences(self, intervals) -> EncodedRaggedArray:
        """indexed_fasta.py:165-206: ``intervals`` has .chromosome (names), .start, .stop (or is an iterable of
        (chromosome, start, stop)).  Every interval is gathered on the device with one synchronisation, for the
        output size.  Intervals on the device (an Interval or Bed6 chunk) have their names looked up there: an
        interval outside its contig raises ValueError and an unknown chromosome KeyError.  Host intervals are
        uploaded once: an unknown chromosome raises KeyError, an interval outside its contig or the file
        AssertionError.  An interval holds at most INT32_MAX bases, as row lengths are int32; a longer one is reported
        like one outside its contig (fa[name] goes in pieces and has no such limit)."""
        contig_ids, text, name_offsets, contigs = self._name_table()
        on_device = _on_device(intervals)
        if on_device:
            rows = RowView(intervals.chromosome)
            start, stop = intervals.start.to(torch.int64).contiguous(), intervals.stop.to(torch.int64).contiguous()
            ids, st_names = ops.name_lookup(rows.base, rows.starts, rows.lens, text, name_offsets)
            bad_names = [st_names[nv.ST_BAD_BASE:nv.ST_BAD_BASE + 1]]
            name_of = lambda r: intervals.chromosome[r].to_string()
        else:
            if hasattr(intervals, "chromosome"):
                intervals = zip(intervals.chromosome, intervals.start, intervals.stop)
            rows = [(c if isinstance(c, str) else c.to_string(), int(a), int(b)) for c, a, b in intervals]
            name_of = lambda r: rows[r][0]
            cols = torch.tensor([[contig_ids[n] for n, _, _ in rows], [a for _, a, _ in rows], [b for _, _, b in rows]],
                                dtype=torch.int64).to(self._file.device)
            ids, start, stop, bad_names = cols[0].to(torch.int32), cols[1], cols[2], []
        out, row_lens, bad_row, bad_name = ops.interval_gather(self._file, start, stop, ids, contigs, extra=bad_names)
        if bad_name and bad_name[0] != nv.INT64_MAX:
            raise KeyError(name_of(bad_name[0]))
        if bad_row is not None:
            name = name_of(bad_row)
            where = f"interval {bad_row} ({name}:{int(start[bad_row])}-{int(stop[bad_row])})"
            rlen = self._index[name]["rlen"]
            if on_device:
                raise ValueError(f"{where} is not inside the contig ({rlen} bases)")
            raise AssertionError(f"{where} reaches beyond the file or its contig ({rlen} bases)")
        return EncodedRaggedArray(EncodedArray(out, BaseEncoding), row_lens)


def _on_device(intervals):
    """Whether ``intervals`` is a record chunk whose chromosome, start and stop already live on the device, so that
    the names are looked up there; anything else is read on the host and uploaded."""
    chrom = getattr(intervals, "chromosome", None)
    start, stop = getattr(intervals, "start", None), getattr(intervals, "stop", None)
    return (isinstance(chrom, EncodedRaggedArray) and chrom.device.type == "cuda" and
            all(isinstance(t, torch.Tensor) and t.is_cuda for t in (start, stop)))


def open_indexed(filename) -> IndexedFasta:
    """io/indexed_files.py:16-37: an IndexedFasta of ``filename`` (its .fai next to it, else built)."""
    return IndexedFasta(filename)
