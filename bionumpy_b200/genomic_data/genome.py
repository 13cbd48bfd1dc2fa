"""Genome, GenomicIntervals and GenomicArray on the device (mirror of bionumpy/genomic_data/genome.py:19-261,
genomic_intervals.py and genomic_track.py, for in-memory data).

A genome lays its contigs end to end in file order: a contig's first position is the sum of the sizes before it
(GenomicArrayGlobal).  Intervals are kept with their global start and stop, so a pileup of every contig is one sort
and one run pass, and a track is one run-length array in global coordinates, split into contigs on demand."""
import os
from pathlib import PurePath

import numpy as np
import torch

from .. import _native as nv
from .. import ops
from ..arithmetics.intervals import (GenomicRunLengthArray, RunsRaggedArray, _add_operators, _device, _int64,
                                     coverage_runs, to_device, track_ufunc)
from ..datatypes import BedGraph, Interval, replace
from ..encoded_array import BaseEncoding, EncodedArray, EncodedRaggedArray
from ..rows import RowView


def ignore_underscores(name):
    """genome_context.py:18-19: contigs whose name holds '_' (alternative haplotypes, unplaced scaffolds) are left out."""
    return "_" not in name


def keep_all(name):
    return True


class Genome:
    """Contig names and sizes in file order (genome.py:19-37).  Contigs the filter rejects are known but left out:
    intervals on them are dropped.  ``filter_function=None`` keeps every contig (genome_context.py:92-93)."""

    def __init__(self, chrom_sizes, fasta_filename=None, sort_names=False, filter_function=keep_all):
        if sort_names:
            chrom_sizes = {key: chrom_sizes[key] for key in sorted(chrom_sizes)}
        self._all = {str(k): int(v) for k, v in chrom_sizes.items()}
        self._sizes = {k: v for k, v in self._all.items() if filter_function is None or filter_function(k)}
        ends = np.cumsum([0] + list(self._sizes.values())).astype(np.int64)
        self._offsets = dict(zip(self._sizes, ends[:-1].tolist()))
        self.size = int(ends[-1])
        self._fasta_filename = fasta_filename
        self._table = None
        self._layout_cache = None

    @classmethod
    def from_dict(cls, chrom_sizes, *args, **kwargs) -> "Genome":
        """genome.py:54-76.

        >>> Genome.from_dict({'chr1': 1000, 'chr2': 2000})
        Genome(['chr1', 'chr2'])"""
        return cls(chrom_sizes, *args, **kwargs)

    @classmethod
    def from_file(cls, filename, sort_names=False, filter_function=ignore_underscores) -> "Genome":
        """genome.py:78-116: a .chrom.sizes or .fai file (name and size in the first two columns), or a .fa / .fasta
        file, whose index is built in memory (no .fai is written)."""
        path = PurePath(filename)
        fasta = None
        if path.suffix in (".fa", ".fasta"):
            fasta = str(filename)
            fai = str(filename) + ".fai"
            if os.path.isfile(fai):
                sizes = _read_sizes(fai)
            else:
                from ..io.indexed_fasta import create_index
                sizes = {name: v["rlen"] for name, v in create_index(filename).items()}
        else:
            sizes = _read_sizes(filename)
        return cls(sizes, fasta_filename=fasta, sort_names=sort_names, filter_function=filter_function)

    def get_chromosome_sizes(self):
        return dict(self._sizes)

    @property
    def chrom_sizes(self):
        return dict(self._sizes)

    def __repr__(self):
        names = list(self._sizes)
        return f"Genome({names[:10] + ['...'] * (len(names) > 10)})"

    def _name_table(self):
        """Every known name sorted as bytes (for bnpk_name_lookup) and, per name in that order, its global offset (-1
        for a contig that is left out) and size; built once on the device."""
        if self._table is None:
            dev = _device()
            names = sorted(self._all, key=lambda n: n.encode())
            raw = [n.encode() for n in names]
            ends = np.cumsum([0] + [len(b) for b in raw]).astype(np.int64)
            text = to_device(np.frombuffer(b"".join(raw) or b"\0", dtype=np.uint8), dev)
            offset = to_device(np.array([self._offsets.get(n, -1) for n in names], dtype=np.int64), dev)
            size = to_device(np.array([self._all[n] for n in names], dtype=np.int64), dev)
            self._table = (names, text, to_device(ends, dev), offset, size)
        return self._table

    def _layout(self):
        """The contigs a track's rows can lie on: the kept contigs of size > 0 in genome order, as their global ends
        (int64[C + 1], from 0) and their indices in the name table (int64[C]); built once on the device."""
        if self._layout_cache is None:
            names = self._name_table()[0]
            index = {n: i for i, n in enumerate(names)}
            kept = [n for n, size in self._sizes.items() if size > 0]
            ends = np.cumsum([0] + [self._sizes[n] for n in kept]).astype(np.int64)
            dev = self._name_table()[1].device
            self._layout_cache = (to_device(ends, dev), to_device(np.array([index[n] for n in kept], dtype=np.int64), dev))
        return self._layout_cache

    def _rows(self, track, mode):
        """The rows of a global track (bnpk_runs_to_intervals, one synchronisation): (name table index int64, global
        start, global stop, value or None), each cut at the contig borders."""
        ends, name_ids = self._layout()
        dev = ends.device
        if name_ids.numel() == 0:
            empty = torch.zeros(0, dtype=torch.int64, device=dev)
            return empty, empty, empty, empty if mode == nv.RUNS_TO_ALL else None
        contig, start, stop, value, n_out = ops.runs_to_intervals(track._events, track._values64(), ends, mode)
        k = int(n_out.cpu()[0])
        value = None if value is None else value[:k]
        return name_ids[contig[:k].to(torch.int64)], start[:k], stop[:k], value

    def _names_of(self, ids):
        """The names of name-table rows ``ids`` (int64) as text views into the device name table, no copy."""
        _, text, name_offsets, _, _ = self._name_table()
        lens = (name_offsets[1:] - name_offsets[:-1])[ids].to(torch.int32)
        return EncodedRaggedArray(EncodedArray(text, BaseEncoding), lens, starts=name_offsets[ids])

    def get_intervals(self, intervals, stranded=False) -> "GenomicIntervals":
        """genome.py:181-209: the intervals of a record (Interval, Bed6, ...) placed on this genome."""
        return GenomicIntervals.from_intervals(intervals, self)

    def read_intervals(self, filename, stranded=False, stream=False, buffer_type=None) -> "GenomicIntervals":
        """genome.py:211-261: a BED file, or the alignments of a BAM file (BamIntervalBuffer), read on the device and
        placed on this genome (stream=False only)."""
        if stream:
            raise NotImplementedError("streamed genomes are not supported")
        from ..io.files import bnp_open, _suffix
        if buffer_type is None and _suffix(str(filename))[0] == ".bam":
            from ..io.bam import BamIntervalBuffer       # genome.py:258-259: alignments as intervals
            buffer_type = BamIntervalBuffer
        if buffer_type is None and stranded:
            from ..io.delimited import Bed6Buffer
            buffer_type = Bed6Buffer
        return self.get_intervals(bnp_open(filename, buffer_type=buffer_type).read(), stranded)


def _read_sizes(filename):
    out = {}
    for line in open(filename):
        parts = line.split()
        if len(parts) >= 2:
            out[parts[0]] = int(parts[1])
    return out


class GenomicIntervals:
    """Intervals on a genome (genomic_intervals.py): the record, each row's contig (an index of the genome's sorted
    name table) and its global start and stop, all on the device."""

    def __init__(self, record, ids, g_start, g_stop, genome):
        self._record, self._ids, self._g_start, self._g_stop, self._genome = record, ids, g_start, g_stop, genome

    @classmethod
    def from_intervals(cls, record, genome):
        """The rows' names are looked up on the device.  An unknown name raises KeyError; an interval with start < 0,
        stop < start or stop past its contig raises ValueError naming the first one; rows on contigs the genome
        leaves out are dropped."""
        names, text, name_offsets, offset, size = genome._name_table()
        dev = text.device
        rows = RowView(record.chromosome)
        start, stop = _int64(record.start, dev), _int64(record.stop, dev)
        ids, st_names = ops.name_lookup(rows.base, rows.starts, rows.lens, text, name_offsets)
        _, g_start, g_stop, st_rows = ops.interval_events(start, stop, ids, offset, size, keys=False, glob=True)
        keep = offset[ids.clamp(min=0).to(torch.int64)] >= 0
        unknown, bad, n_keep = torch.cat([st_names[nv.ST_BAD_BASE:nv.ST_BAD_BASE + 1],
                                          st_rows[nv.ST_BAD_BASE:nv.ST_BAD_BASE + 1],
                                          keep.sum().reshape(1)]).cpu().tolist()
        if unknown != nv.INT64_MAX:
            raise KeyError(record.chromosome[unknown].to_string())
        if bad != nv.INT64_MAX:
            name = record.chromosome[bad].to_string()
            raise ValueError(f"interval {bad} ({name}:{int(start[bad])}-{int(stop[bad])}) is not inside the contig "
                             f"({genome._all[name]} bases)")
        out = cls(record, ids, g_start, g_stop, genome)
        if n_keep < len(ids):
            out = out[torch.nonzero(keep).reshape(-1)]
        return out

    @classmethod
    def from_track(cls, track) -> "GenomicIntervals":
        """The intervals where a GenomicArray is not 0 (genomic_intervals.py:529-543), in genome order, cut at contig
        borders; one synchronisation.  Neighbouring non-zero runs are one interval whatever their values.  The
        reference returns every run of an integer track as a bedGraph here, against its own docstring; this follows
        the docstring."""
        genome = track._genome
        ids, g_start, g_stop, _ = genome._rows(track._global, nv.RUNS_TO_NONZERO)
        offset = genome._name_table()[3]
        record = Interval(genome._names_of(ids), g_start - offset[ids], g_stop - offset[ids])
        return cls(record, ids.to(torch.int32), g_start, g_stop, genome)

    @property
    def chromosome(self):
        return self._record.chromosome

    @property
    def start(self):
        return self._record.start

    @property
    def stop(self):
        return self._record.stop

    def get_data(self):
        return self._record

    def __len__(self):
        return self._ids.numel()

    def __getitem__(self, idx):
        """The selected intervals (a bool mask, an index tensor/array/list)."""
        if isinstance(idx, (list, np.ndarray)):
            idx = torch.as_tensor(np.asarray(idx))
        if isinstance(idx, torch.Tensor):
            idx = idx.to(self._ids.device)
        return GenomicIntervals(self._record[idx], self._ids[idx], self._g_start[idx], self._g_stop[idx], self._genome)

    def __repr__(self):
        names = list(self._genome._sizes)
        return f"Genomic Intervals on {names[:10] + ['...'] * (len(names) > 10)}:\n{self._record!r}"

    def _runs(self, mode):
        runs, values, bad = coverage_runs(self._g_start, self._g_stop, self._genome.size, mode)
        assert bad is None      # every row was checked against its contig when the intervals were made
        return GenomicArray(runs, values if mode == nv.PILEUP_COUNT else values.to(torch.bool), self._genome)

    def get_pileup(self) -> "GenomicArray":
        """The number of intervals that cover each position of the genome: one sort and one run pass for every contig,
        one synchronisation."""
        return self._runs(nv.PILEUP_COUNT)

    def get_mask(self) -> "GenomicArray":
        """Where any interval covers the genome (bool)."""
        return self._runs(nv.PILEUP_ANY)

    def sorted(self) -> "GenomicIntervals":
        """The intervals in genome order, then by start, then by stop, stably (genomic_intervals.py:691-699); on the
        device, no synchronisation."""
        from ..arithmetics.intervals import lexsort_order
        names = self._genome._name_table()[0]
        order = {n: i for i, n in enumerate(self._genome._sizes)}
        rank = to_device(np.array([order.get(n, -1) for n in names], dtype=np.int64), self._ids.device)
        return self[lexsort_order(self._g_stop, self._g_start, rank[self._ids.to(torch.int64)])]

    def merged(self, distance=0) -> "GenomicIntervals":
        """merge_intervals on every contig, in genome order: the rows are sorted by global start on the device, a
        merge never crosses a contig, one synchronisation."""
        if len(self) == 0:
            return self
        order = torch.sort(self._g_start, stable=True).indices
        g_start, g_stop, ids = self._g_start[order], self._g_stop[order], self._ids[order]
        same = torch.cat([torch.zeros(1, dtype=torch.bool, device=ids.device), ids[1:] == ids[:-1]]).to(torch.uint8)
        first, stops, n_out, _ = ops.interval_merge(g_start, g_stop, same, distance)
        k = int(n_out.cpu()[0])
        first = first[:k]
        sel = order[first]
        record = self._record[sel]
        local = stops[:k] - g_start[first] + _int64(record.start, ids.device)
        return GenomicIntervals(replace(record, stop=local), ids[first], g_start[first], stops[:k], self._genome)


class GenomicArray:
    """A track over a whole genome (GenomicArrayGlobal): one run-length array in global coordinates on the device."""

    def __init__(self, events, values, genome):
        self._global = GenomicRunLengthArray(events, values, genome.size)
        self._genome = genome

    @classmethod
    def _of(cls, track, genome):
        out = cls.__new__(cls)
        out._global, out._genome = track, genome
        return out

    @property
    def dtype(self):
        return self._global.dtype

    def __array_ufunc__(self, ufunc, method, *inputs, **kwargs):
        """Track operators and the ufuncs of arithmetics.intervals.TRACK_UFUNCS between tracks on genomes with the
        same contigs and sizes (else ValueError) and integer or bool scalars, on the runs (one synchronisation); any
        other call gets the dense arrays of the whole genome."""
        genomes = [x._genome for x in inputs if isinstance(x, GenomicArray)]
        for g in genomes[1:]:
            if list(g._sizes.items()) != list(genomes[0]._sizes.items()):
                raise ValueError("the tracks are on genomes with different contigs or sizes")
        args = [x._global if isinstance(x, GenomicArray) else x for x in inputs]
        out = track_ufunc(ufunc, method, args, kwargs)
        if out is None:
            return getattr(ufunc, method)(*[np.asarray(x) if isinstance(x, GenomicRunLengthArray) else x
                                            for x in args], **kwargs)
        return GenomicArray._of(out, genomes[0])

    def __getitem__(self, idx):
        """``track["chr1"]``: one contig's runs.  ``track[intervals]`` (GenomicIntervals, or a record placed on the
        genome here): the lazy per-interval values, one row per interval.  A record with rows on contigs the genome
        leaves out raises ValueError, since those rows would be dropped and the rows would no longer line up with the
        record; place it with genome.get_intervals first to drop them."""
        if isinstance(idx, str):
            return self._contig(idx)
        if not isinstance(idx, GenomicIntervals):
            placed = self._genome.get_intervals(idx)
            if len(placed) != len(idx):
                raise ValueError(f"{len(idx) - len(placed)} of the {len(idx)} intervals are on contigs the genome leaves "
                                 "out; index the track with genome.get_intervals(intervals) to drop them")
            idx = placed
        return RunsRaggedArray(self._global, idx._g_start, idx._g_stop)

    def _contig(self, name):
        """The contig's runs, split off on the device: the run that holds its first position and every run that starts
        inside it, clipped to it."""
        off, size = self._genome._offsets[name], self._genome._sizes[name]
        runs = self._global.starts
        q = torch.tensor([off, off + size], dtype=torch.int64, device=runs.device)
        i0 = torch.searchsorted(runs, q[:1], right=True) - 1
        i1 = torch.searchsorted(runs, q[1:])
        i0, i1 = torch.cat([i0, i1]).cpu().tolist()
        i1 = max(i1, i0 + 1)
        events = (self._global._events[i0:i1 + 1] - off).clamp_(0, size)
        return GenomicRunLengthArray(events, self._global.values[i0:i1], size)

    def to_dict(self):
        return {name: self._contig(name) for name in self._genome._sizes}

    def get_data(self):
        """genomic_track.py:199-218: a bool track as the Interval rows where it is True (GenomicIntervals.from_track),
        any other track as a BedGraph of every run, cut at contig borders, with the track's values; one
        synchronisation."""
        if self.dtype == torch.bool:
            return GenomicIntervals.from_track(self).get_data()
        genome = self._genome
        ids, g_start, g_stop, value = genome._rows(self._global, nv.RUNS_TO_ALL)
        offset = genome._name_table()[3]
        return BedGraph(genome._names_of(ids), g_start - offset[ids], g_stop - offset[ids], self._global._cast(value))

    def sum(self, axis=None, **kwargs):
        return self._global.sum()

    def __repr__(self):
        names = list(self._genome._sizes)
        lines = [f"{name}: {self._contig(name)}" for name in names[:10]]
        if len(names) > 10:
            lines.append("...")
        return "\n".join(lines)


_add_operators(GenomicArray)

__all__ = ["Genome", "GenomicIntervals", "GenomicArray", "ignore_underscores", "keep_all"]
