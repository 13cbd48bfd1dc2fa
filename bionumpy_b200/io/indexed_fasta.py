"""IndexedFasta on the device (mirror of bionumpy/io/indexed_fasta.py:13-206).

The FASTA file is brought to the device once (pinned, prefetching ingest); a contig or a set of intervals is then a
gather that skips the line ends (bnpk_fasta_gather) -- where the reference seeks and reads per interval and deletes the
newline bytes on the host (indexed_fasta.py:101-131, 133-206).  The index is the .fai next to the file (read_index,
indexed_fasta.py:13-31); without one it is built from the file image (create_index, :34-58: name, length, offset of the
first base, bases per line, bytes per line)."""
import os
from pathlib import Path

import numpy as np
import torch

from .. import _native as nv
from .. import config, ops
from ..encoded_array import EncodedArray, EncodedRaggedArray, BaseEncoding
from ..rows import RowView


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

    def _gather(self, names, starts, lens):
        dev = self._file.device
        idx = [self._index[n] for n in names]
        t = lambda v, dt: torch.tensor(v, dtype=dt, device=dev)
        row_len = t(lens, torch.int64)
        offsets = torch.zeros(len(idx) + 1, dtype=torch.int64, device=dev)
        offsets[1:] = torch.cumsum(row_len, 0)
        out = torch.empty(int(sum(lens)), dtype=torch.uint8, device=dev)
        status = nv.new_status(dev)
        # (the argument tensors stay referenced until the launch is queued)
        c_off, r_start = t([i["offset"] for i in idx], torch.int64), t(starts, torch.int64)
        lenc, lenb = t([max(i["lenc"], 1) for i in idx], torch.int32), t([max(i["lenb"], 1) for i in idx], torch.int32)
        nv.check(nv.lib().bnpk_fasta_gather(nv.ptr(self._file), self._file.numel(), len(idx), nv.ptr(c_off), nv.ptr(r_start),
                                            nv.ptr(row_len), nv.ptr(lenc), nv.ptr(lenb), nv.ptr(offsets), nv.ptr(out),
                                            nv.ptr(status), nv.stream_ptr()))
        bad = ops.read_status(status).bad_base()
        assert bad is None, f"interval {bad[0]} reaches beyond the file"
        return out, row_len

    def __getitem__(self, chromosome: str) -> EncodedArray:
        """The whole sequence of a contig (indexed_fasta.py:101-131)."""
        out, _ = self._gather([chromosome], [0], [self._index[chromosome]["rlen"]])
        return EncodedArray(out, BaseEncoding)

    def _name_table(self):
        """The contig names sorted as bytes, concatenated on the device with their offsets, and each contig's
        (offset, lenc, lenb, length) in that order: built once, for bnpk_name_lookup and bnpk_interval_gather."""
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
            self._table = (names, text, torch.from_numpy(ends).to(dev), contigs)
        return self._table

    def get_interval_sequences(self, intervals) -> EncodedRaggedArray:
        """indexed_fasta.py:165-206: ``intervals`` has .chromosome (names), .start, .stop (or is an iterable of
        (chromosome, start, stop)).  Intervals on the device (an Interval or Bed6 chunk) are looked up and gathered
        on the device with one synchronisation, for the output size; an interval outside its contig raises
        ValueError and an unknown chromosome KeyError."""
        if _on_device(intervals):
            return self._device_interval_sequences(intervals)
        if hasattr(intervals, "chromosome"):
            names = [c if isinstance(c, str) else c.to_string() for c in intervals.chromosome]
            starts = [int(x) for x in intervals.start]
            stops = [int(x) for x in intervals.stop]
        else:
            names, starts, stops = zip(*[(c, int(a), int(b)) for c, a, b in intervals])
        lens = [b - a for a, b in zip(starts, stops)]
        out, row_len = self._gather(list(names), list(starts), lens)
        return EncodedRaggedArray(EncodedArray(out, BaseEncoding), row_len.to(torch.int32))

    def _device_interval_sequences(self, intervals):
        names, text, name_offsets, contigs = self._name_table()
        rows = RowView(intervals.chromosome)
        start, stop = intervals.start.to(torch.int64).contiguous(), intervals.stop.to(torch.int64).contiguous()
        ids, st_names = ops.name_lookup(rows.base, rows.starts, rows.lens, text, name_offsets)
        row_lens, st_rows = ops.interval_check(self._file, start, stop, ids, contigs)
        offsets = ops.row_offsets(row_lens)
        total, bad_name, bad_row = (int(x) for x in torch.cat(
            [offsets[-1:], st_names[nv.ST_BAD_BASE:nv.ST_BAD_BASE + 1], st_rows[nv.ST_BAD_BASE:nv.ST_BAD_BASE + 1]]
        ).cpu().tolist())
        if bad_name != nv.INT64_MAX:
            raise KeyError(intervals.chromosome[bad_name].to_string())
        if bad_row != nv.INT64_MAX:
            name = intervals.chromosome[bad_row].to_string()
            raise ValueError(f"interval {bad_row} ({name}:{int(start[bad_row])}-{int(stop[bad_row])}) is not inside "
                             f"the contig ({self._index[name]['rlen']} bases)")
        out = ops.interval_copy(self._file, start, stop, offsets, total, ids, contigs)
        return EncodedRaggedArray(EncodedArray(out, BaseEncoding), row_lens)


def _on_device(intervals):
    """Whether ``intervals`` is a record chunk whose chromosome, start and stop already live on the device."""
    chrom = getattr(intervals, "chromosome", None)
    start, stop = getattr(intervals, "start", None), getattr(intervals, "stop", None)
    return (isinstance(chrom, EncodedRaggedArray) and chrom.device.type == "cuda" and
            all(isinstance(t, torch.Tensor) and t.is_cuda for t in (start, stop)))


def open_indexed(filename) -> IndexedFasta:
    """io/indexed_files.py:16-37: an IndexedFasta of ``filename`` (its .fai next to it, else built)."""
    return IndexedFasta(filename)
