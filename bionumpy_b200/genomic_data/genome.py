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
from ..arithmetics.intervals import (FloatRunLengthArray, GenomicRunLengthArray, RunsRaggedArray, _add_operators,
                                     _device, _int64, _rtruediv, _truediv, coverage_runs, to_device, track_ufunc)
from ..datatypes import BedGraph, Interval, LocationEntry, StrandedInterval, StrandedLocationEntry, replace
from ..encoded_array import BaseEncoding, EncodedArray, EncodedRaggedArray
from ..encodings import StrandEncoding
from ..rows import RowView

MINUS = 1           # StrandEncoding's code of '-' ('+' 0, '.' 2)


def _strand_codes(strand, device):
    """StrandEncoding codes (uint8, on the device) of a record's strand field."""
    codes = strand.raw() if isinstance(strand, EncodedArray) else torch.as_tensor(np.asarray(strand))
    return codes.reshape(-1).to(device, torch.uint8)


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
        """genome.py:181-209: the intervals of a record (Interval, Bed6, ...) placed on this genome.  ``stranded=True``
        keeps the record's strand (a record without a strand field raises ValueError): windows on '-' rows are then
        read back to front when they index a track."""
        return GenomicIntervals.from_intervals(intervals, self, stranded)

    def get_locations(self, entries) -> "GenomicLocation":
        """genome.py:328-349: LocationEntry (or StrandedLocationEntry) records placed on this genome, as
        from_intervals places intervals: an unknown name raises KeyError, a position outside [0, contig size) raises
        ValueError naming the row, and rows on contigs the genome leaves out are dropped.  A strand field makes the
        locations stranded.  One synchronisation.

        >>> genome = Genome.from_dict({'chr1': 100, 'chr2': 50})
        >>> genome.get_locations(LocationEntry(['chr1', 'chr2'], [10, 49])).position.tolist()
        [10, 49]"""
        names, text, name_offsets, offset, size = self._name_table()
        dev = text.device
        rows = RowView(entries.chromosome)
        pos = _int64(entries.position, dev)
        ids, st_names = ops.name_lookup(rows.base, rows.starts, rows.lens, text, name_offsets)
        _, g_pos, _, st_rows = ops.interval_events(pos, pos + 1, ids, offset, size, keys=False, glob=True)
        keep = offset[ids.clamp(min=0).to(torch.int64)] >= 0
        st_names, st_rows, n_keep = ops.read_back(st_names, st_rows, keep.sum())
        if st_names.fault is not None:
            raise KeyError(entries.chromosome[st_names.fault].to_string())
        bad = st_rows.fault
        if bad is not None:
            name = entries.chromosome[bad].to_string()
            raise ValueError(f"location {bad} ({name}:{int(pos[bad])}) is not inside the contig "
                             f"({self._all[name]} bases)")
        strand = _strand_codes(entries.strand, dev) if "strand" in entries._fields else None
        out = GenomicLocation(ids.to(torch.int64), g_pos, pos, self, strand)
        if n_keep < len(ids):
            out = out[torch.nonzero_static(keep, size=n_keep).reshape(-1)]
        return out

    def _rank(self, ids):
        """The genome-order rank of every row's contig (ids index the name table; left-out contigs rank -1)."""
        names = self._name_table()[0]
        order = {n: i for i, n in enumerate(self._sizes)}
        rank = to_device(np.array([order.get(n, -1) for n in names], dtype=np.int64), ids.device)
        return rank[ids.to(torch.int64)]

    def read_intervals(self, filename, stranded=False, stream=False, buffer_type=None) -> "GenomicIntervals":
        """genome.py:211-261: a BED file, or the alignments of a BAM or SAM file (BamIntervalBuffer, SAMIntervalBuffer),
        read on the device and placed on this genome (stream=False only)."""
        if stream:
            raise NotImplementedError("streamed genomes are not supported")
        from ..io.files import bnp_open, _suffix
        suffix = _suffix(str(filename))[0]
        if buffer_type is None and suffix == ".bam":
            from ..io.bam import BamIntervalBuffer       # genome.py:258-259: alignments as intervals
            buffer_type = BamIntervalBuffer
        if buffer_type is None and suffix == ".sam":
            from ..io.sam import SAMIntervalBuffer
            buffer_type = SAMIntervalBuffer
        if buffer_type is None and stranded:
            from ..io.delimited import Bed6Buffer
            buffer_type = Bed6Buffer
        return self.get_intervals(bnp_open(filename, buffer_type=buffer_type).read(), stranded)

    def get_track(self, bedgraph) -> "GenomicArray":
        """genome.py:127-152: the GenomicArray of BedGraph rows, placed as GenomicIntervals.from_intervals places
        intervals (an unknown name raises KeyError, a row with stop < start or past its contig ValueError naming it, and
        rows on contigs the genome leaves out are dropped).  The rows may come in any order: they are sorted by global
        start on the device.  Rows that overlap raise ValueError naming the first pair (the reference assumes sorted,
        disjoint rows).  Empty rows add nothing; the positions no row covers are +0.0; neighbouring runs whose values
        are bitwise equal are one run.  Float values give a float track, integer or bool values an integer or bool one.

        The lookup, bounds, overlap check and run count are read back in one synchronisation; the library launches
        two kernels (the name lookup and the bounds check), the runs are built by torch ops.

        >>> bedgraph = BedGraph(['chr1', 'chr1', 'chr2'], [0, 10, 0], [5, 15, 5], [1, 2, 3])
        >>> Genome.from_dict({'chr1': 20, 'chr2': 10}).get_track(bedgraph)
        chr1: [1 1 1 1 1 0 0 0 0 0 2 2 2 2 2 0 0 0 0 0]
        chr2: [3 3 3 3 3 0 0 0 0 0]"""
        names, text, name_offsets, offset, size = self._name_table()
        dev, G = text.device, self.size
        value = bedgraph.value if isinstance(bedgraph.value, torch.Tensor) else torch.as_tensor(np.asarray(bedgraph.value))
        value = value.to(dev)
        is_float = value.is_floating_point()
        bits = value.to(torch.float64).view(torch.int64) if is_float else value.to(torch.int64)
        zero = torch.zeros(1, dtype=torch.int64, device=dev)
        start, stop = _int64(bedgraph.start, dev), _int64(bedgraph.stop, dev)
        if start.numel() == 0 or G == 0:
            events = torch.cat([zero, torch.full((1,), G, dtype=torch.int64, device=dev)])
            return self._track_of(events, zero, value.dtype)
        rows = RowView(bedgraph.chromosome)
        ids, st_names = ops.name_lookup(rows.base, rows.starts, rows.lens, text, name_offsets)
        _, g_start, g_stop, st_rows = ops.interval_events(start, stop, ids, offset, size, keys=False, glob=True)
        keep = (offset[ids.clamp(min=0).to(torch.int64)] >= 0) & (g_stop > g_start)
        # the kept rows by global start, then every other row as an empty row at the end, then one more: row i
        # contributes the gap [e[i - 1], s[i]) of +0.0 and its own run [s[i], e[i])
        end = torch.full((1,), G, dtype=torch.int64, device=dev)
        order = torch.sort(torch.where(keep, g_start, G), stable=True).indices
        s = torch.cat([torch.where(keep, g_start, G)[order], end])
        e = torch.cat([torch.where(keep, g_stop, G)[order], end])
        v = torch.cat([bits[order], zero])
        prev_e, prev_v = torch.cat([zero, e[:-1]]), torch.cat([zero, v[:-1]])
        index = torch.arange(s.numel(), dtype=torch.int64, device=dev)
        first_overlap = torch.where(prev_e > s, index, s.numel()).min().reshape(1)       # s.numel(): none
        first, gap = index == 0, s > prev_e
        # a run starts where the value's bits differ from those of the non-empty piece before it
        emit_gap = gap & (first | (prev_v != 0))
        emit_row = (e > s) & torch.where(gap, v != 0, first | (v != prev_v))
        emit = torch.stack([emit_gap, emit_row], 1).reshape(-1)
        st_names, st_rows, n_runs, bad = ops.read_back(st_names, st_rows, emit.sum(), first_overlap)
        if st_names.fault is not None:
            raise KeyError(bedgraph.chromosome[st_names.fault].to_string())
        if st_rows.fault is not None:
            row = st_rows.fault
            name = bedgraph.chromosome[row].to_string()
            raise ValueError(f"bedGraph row {row} ({name}:{int(start[row])}-{int(stop[row])}) is not inside the "
                             f"contig ({self._all[name]} bases)")
        if bad < s.numel():
            a, b = order[bad - 1:bad + 1].cpu().tolist()
            raise ValueError(f"bedGraph rows {a} and {b} overlap: {bedgraph.chromosome[a].to_string()}:"
                             f"{int(start[a])}-{int(stop[a])} and {bedgraph.chromosome[b].to_string()}:"
                             f"{int(start[b])}-{int(stop[b])}")
        picked = torch.nonzero_static(emit, size=n_runs).reshape(-1)
        run_starts = torch.stack([prev_e, s], 1).reshape(-1)[picked]
        run_bits = torch.stack([torch.zeros_like(v), v], 1).reshape(-1)[picked]
        return self._track_of(torch.cat([run_starts, end]), run_bits, value.dtype)

    def _track_of(self, events, bits, dtype):
        """A GenomicArray of runs whose values are int64 (their bits, for a float dtype)."""
        if dtype.is_floating_point:
            return GenomicArray._of(FloatRunLengthArray(events, bits.view(torch.float64), self.size), self)
        values = bits != 0 if dtype == torch.bool else bits
        return GenomicArray._of(GenomicRunLengthArray(events, values, self.size), self)

    def read_track(self, filename, stream=False) -> "GenomicArray":
        """genome.py:154-179: a bedGraph file (.bdg, .bdg.gz) read on the device and made a GenomicArray by get_track
        (stream=False only)."""
        if stream:
            raise NotImplementedError("streamed genomes are not supported")
        from ..io.files import bnp_open
        return self.get_track(bnp_open(filename).read())

    def read_annotation(self, filename) -> "GenomicAnnotation":
        """genome.py:390-422: a GTF or GFF file read on the device, with its genes, transcripts and exons placed on
        this genome when first asked for (rows on contigs the genome leaves out are dropped)."""
        from ..io.files import bnp_open
        return GenomicAnnotation(bnp_open(filename).read(), self)


def _read_sizes(filename):
    out = {}
    for line in open(filename):
        parts = line.split()
        if len(parts) >= 2:
            out[parts[0]] = int(parts[1])
    return out


class GenomicIntervals:
    """Intervals on a genome (genomic_intervals.py): the record, each row's contig (an index of the genome's sorted
    name table) and its global start and stop, all on the device.  Stranded intervals also carry each row's strand
    (StrandEncoding codes); a track indexed by them gives the values of '-' rows back to front."""

    def __init__(self, record, ids, g_start, g_stop, genome, strand=None):
        self._record, self._ids, self._g_start, self._g_stop, self._genome = record, ids, g_start, g_stop, genome
        self._strand = strand

    @classmethod
    def from_intervals(cls, record, genome, stranded=False):
        """The rows' names are looked up on the device.  An unknown name raises KeyError; an interval with start < 0,
        stop < start or stop past its contig raises ValueError naming the first one; rows on contigs the genome
        leaves out are dropped.  ``stranded=True`` keeps the record's strand; a record without one raises
        ValueError."""
        if stranded and "strand" not in record._fields:
            raise ValueError(f"stranded intervals need a strand field, which {type(record).__name__} has not")
        names, text, name_offsets, offset, size = genome._name_table()
        dev = text.device
        rows = RowView(record.chromosome)
        start, stop = _int64(record.start, dev), _int64(record.stop, dev)
        ids, st_names = ops.name_lookup(rows.base, rows.starts, rows.lens, text, name_offsets)
        _, g_start, g_stop, st_rows = ops.interval_events(start, stop, ids, offset, size, keys=False, glob=True)
        keep = offset[ids.clamp(min=0).to(torch.int64)] >= 0
        st_names, st_rows, n_keep = ops.read_back(st_names, st_rows, keep.sum())
        if st_names.fault is not None:
            raise KeyError(record.chromosome[st_names.fault].to_string())
        bad = st_rows.fault
        if bad is not None:
            name = record.chromosome[bad].to_string()
            raise ValueError(f"interval {bad} ({name}:{int(start[bad])}-{int(stop[bad])}) is not inside the contig "
                             f"({genome._all[name]} bases)")
        out = cls(record, ids, g_start, g_stop, genome, _strand_codes(record.strand, dev) if stranded else None)
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

    @property
    def strand(self):
        """The strand of every row; unstranded intervals raise ValueError, as in the reference."""
        if self._strand is None:
            raise ValueError("Unstranded interval has not strand")
        return self._record.strand

    def is_stranded(self) -> bool:
        return self._strand is not None

    def _location_strand(self):
        """The strand codes get_location and extended_to_size go by, or None."""
        return self._strand

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
        strand = None if self._strand is None else self._strand[idx]
        return type(self)(self._record[idx], self._ids[idx], self._g_start[idx], self._g_stop[idx], self._genome,
                          strand)

    def _contig_bounds(self):
        """Each row's contig offset and size (int64 device tensors)."""
        _, _, _, offset, size = self._genome._name_table()
        ids = self._ids.to(torch.int64)
        return offset[ids], size[ids]

    def _with(self, start, stop):
        """These intervals with new local starts and stops, clipped to [0, contig size); the record keeps its type
        and every other field."""
        offset, size = self._contig_bounds()
        start, stop = start.clamp(min=0), torch.minimum(stop, size)
        return type(self)(replace(self._record, start=start, stop=stop), self._ids, offset + start, offset + stop,
                          self._genome, self._strand)

    def clip(self) -> "GenomicIntervals":
        """The intervals clipped to [0, contig size) (genomic_intervals.py:819-830); no synchronisation."""
        offset, _ = self._contig_bounds()
        return self._with(self._g_start - offset, self._g_stop - offset)

    def extended_to_size(self, size: int) -> "GenomicIntervals":
        """Every interval made ``size`` long along its strand (genomic_intervals.py:755-768), then clipped: '+' rows
        keep their start, '-' rows their stop; '.' and unstranded rows behave as '+'.  ``reads.extended_to_size(200)
        .get_pileup()`` is a fragment pileup.  No synchronisation."""
        offset, _ = self._contig_bounds()
        start, stop = self._g_start - offset, self._g_stop - offset
        strand = self._location_strand()
        if strand is None:
            return self._with(start, start + size)
        minus = strand == MINUS
        return self._with(torch.where(minus, stop - size, start), torch.where(minus, stop, start + size))

    def get_location(self, where: str = "start") -> "GenomicLocation":
        """The 'start', 'stop' or 'center' of every interval (genomic_intervals.py:705-733), stranded when the
        intervals are.  On a '-' row 'start' is stop - 1 and 'stop' is start; on '+', '.' and unstranded rows 'start'
        is start and 'stop' is stop - 1; 'center' is (start + stop) // 2.  No synchronisation."""
        if where not in ("start", "stop", "center"):
            raise ValueError(f"where must be 'start', 'stop' or 'center', not {where!r}")
        offset, _ = self._contig_bounds()
        start, stop = self._g_start - offset, self._g_stop - offset
        strand = self._location_strand()
        if where == "center":
            pos = torch.div(start + stop, 2, rounding_mode="floor")
        else:
            first, last = (start, stop - 1) if where == "start" else (stop - 1, start)
            pos = first if strand is None else torch.where(strand == MINUS, last, first)
        return GenomicLocation(self._ids.to(torch.int64), offset + pos, pos, self._genome, strand)

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
        return self[lexsort_order(self._g_stop, self._g_start, self._genome._rank(self._ids))]

    def merged(self, distance=0) -> "GenomicIntervals":
        """merge_intervals on every contig, in genome order: the rows are sorted by global start on the device, a
        merge never crosses a contig, one synchronisation.  The result is unstranded, as in the reference."""
        if len(self) == 0:
            return GenomicIntervals(self._record, self._ids, self._g_start, self._g_stop, self._genome)
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


class Genes(GenomicIntervals):
    """annotation.py Genes: gene intervals with their strand and gene_id.  They always carry a strand, so
    get_location and extended_to_size go by it and give stranded results, as the reference's stranded annotation does;
    a track indexed by the features themselves is read forward on every strand, as before."""

    @property
    def strand(self):
        return self._record.strand

    def is_stranded(self) -> bool:
        return True

    def _location_strand(self):
        return self._strand if self._strand is not None else _strand_codes(self._record.strand, self._ids.device)

    @property
    def gene_id(self):
        return self._record.gene_id


class Transcripts(Genes):
    @property
    def transcript_id(self):
        return self._record.transcript_id


class Exons(Transcripts):
    @property
    def exon_id(self):
        return self._record.exon_id


class GenomicLocation:
    """Positions on a genome (genomic_intervals.py GenomicLocation): each row's contig (an index of the genome's sorted
    name table), its global and local position and, for stranded locations, its strand (StrandEncoding codes), all on
    the device.  Made by Genome.get_locations and GenomicIntervals.get_location."""

    def __init__(self, ids, g_pos, pos, genome, strand=None):
        self._ids, self._g_pos, self._pos, self._genome, self._strand = ids, g_pos, pos, genome, strand

    @property
    def chromosome(self):
        return self._genome._names_of(self._ids)

    @property
    def position(self):
        return self._pos

    @property
    def strand(self):
        if self._strand is None:
            raise ValueError("Unstranded location has not strand")
        return EncodedArray(self._strand, StrandEncoding)

    def is_stranded(self) -> bool:
        return self._strand is not None

    def __len__(self):
        return self._ids.numel()

    def __getitem__(self, idx):
        """The selected locations (a bool mask, an index tensor/array/list)."""
        if isinstance(idx, (list, np.ndarray)):
            idx = torch.as_tensor(np.asarray(idx))
        if isinstance(idx, torch.Tensor):
            idx = idx.to(self._ids.device)
        strand = None if self._strand is None else self._strand[idx]
        return GenomicLocation(self._ids[idx], self._g_pos[idx], self._pos[idx], self._genome, strand)

    def sorted(self) -> "GenomicLocation":
        """The locations in genome order, then by position, stably; on the device, no synchronisation."""
        from ..arithmetics.intervals import lexsort_order
        return self[lexsort_order(self._pos, self._genome._rank(self._ids))]

    def get_data(self):
        """The locations as LocationEntry records, or StrandedLocationEntry when stranded."""
        if self._strand is None:
            return LocationEntry(self.chromosome, self._pos)
        return StrandedLocationEntry(self.chromosome, self._pos, self.strand)

    def get_windows(self, flank=None, window_size=None) -> GenomicIntervals:
        """Windows around the locations (genomic_intervals.py:212-243): [p - flank, p + flank + 1) with ``flank``, else
        [p - window_size // 2, p + window_size // 2 + window_size % 2), clipped to the contig and stranded when the
        locations are.  No synchronisation."""
        if (flank is None) == (window_size is None):
            raise ValueError("give one of flank and window_size")
        left, right = (flank, flank + 1) if flank is not None else (window_size // 2, window_size // 2 + window_size % 2)
        names = self.chromosome
        if self._strand is None:
            record = Interval(names, self._pos - left, self._pos + right)
        else:
            record = StrandedInterval(names, self._pos - left, self._pos + right, self.strand)
        offset = self._g_pos - self._pos
        windows = GenomicIntervals(record, self._ids, offset + record.start, offset + record.stop, self._genome,
                                   self._strand)
        return windows.clip()

    def __repr__(self):
        names = list(self._genome._sizes)
        return f"Genomic Locations on {names[:10] + ['...'] * (len(names) > 10)}: {len(self)} locations"


class GenomicAnnotation:
    """annotation.py GenomicAnnotation: the genes, transcripts and exons of GTF/GFF entries on a genome, each selected
    and placed on the genome the first time it is asked for."""

    def __init__(self, data, genome):
        self._data, self._genome = data, genome
        self._genes = self._transcripts = self._exons = None

    @classmethod
    def from_gtf_entries(cls, gtf_entries, genome) -> "GenomicAnnotation":
        return cls(gtf_entries, genome)

    @property
    def genes(self) -> Genes:
        if self._genes is None:
            self._genes = Genes.from_intervals(self._data.get_genes(), self._genome)
        return self._genes

    @property
    def transcripts(self) -> Transcripts:
        if self._transcripts is None:
            self._transcripts = Transcripts.from_intervals(self._data.get_transcripts(), self._genome)
        return self._transcripts

    @property
    def exons(self) -> Exons:
        if self._exons is None:
            self._exons = Exons.from_intervals(self._data.get_exons(), self._genome)
        return self._exons

    def __repr__(self):
        return f"GenomicAnnotation(genome={self._genome!r}, data={self._data!r})"


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
        genome here): the lazy per-interval values, one row per interval; the rows of stranded intervals on '-' are
        read back to front.  A record with rows on contigs the genome leaves out raises ValueError, since those rows
        would be dropped and the rows would no longer line up with the record; place it with genome.get_intervals first
        to drop them.  ``track[locations]`` (GenomicLocation): the value at every location in the track's dtype, with
        no synchronisation."""
        if isinstance(idx, str):
            return self._contig(idx)
        if isinstance(idx, GenomicLocation):
            track, n = self._global, len(idx)
            offsets = torch.arange(n + 1, dtype=torch.int64, device=idx._g_pos.device)
            return track._cast(ops.runs_extract(track._events, track._values64(), idx._g_pos.contiguous(), offsets, n))
        if not isinstance(idx, GenomicIntervals):
            placed = self._genome.get_intervals(idx)
            if len(placed) != len(idx):
                raise ValueError(f"{len(idx) - len(placed)} of the {len(idx)} intervals are on contigs the genome leaves "
                                 "out; index the track with genome.get_intervals(intervals) to drop them")
            idx = placed
        reverse = None if idx._strand is None else idx._strand == MINUS
        return RunsRaggedArray(self._global, idx._g_start, idx._g_stop, reverse)

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
        return type(self._global)(events, self._global.values[i0:i1], size)

    def to_dict(self):
        return {name: self._contig(name) for name in self._genome._sizes}

    def get_data(self):
        """genomic_track.py:199-218: a bool track as the Interval rows where it is True (GenomicIntervals.from_track),
        any other track as a BedGraph of every run, cut at contig borders, with the track's values (float64 for a
        float track); one synchronisation."""
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
GenomicArray.__truediv__, GenomicArray.__rtruediv__ = _truediv, _rtruediv

__all__ = ["Genome", "GenomicIntervals", "GenomicLocation", "GenomicArray", "GenomicAnnotation", "Genes", "Transcripts",
           "Exons", "ignore_underscores", "keep_all"]
