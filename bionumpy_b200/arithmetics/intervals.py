"""Pileups, masks and merges of intervals on one contig (mirror of bionumpy/arithmetics/intervals.py:19-304).

  get_pileup / get_boolean_mask : every interval becomes two event keys (bnpk_interval_events), torch.sort orders them
                                  and one look-back pass writes the runs of the coverage (bnpk_pileup_runs); one
                                  synchronisation reads the run count and the first bad interval.
  merge_intervals               : the reference's running-max rule as one segmented look-back scan
                                  (bnpk_interval_merge), segments cut where the chromosome name changes
                                  (bnpk_rows_equal_prev); one synchronisation.
  GenomicRunLengthArray         : runs on the device; indexing by intervals gives a lazy ragged result whose per-row
                                  max / min / sum / mean / any run fused over the runs (bnpk_runs_reduce) and whose
                                  values, when asked for, are gathered by bnpk_runs_extract."""
import numpy as np
import torch

from .. import _native as nv
from .. import config, ops
from ..datatypes import replace
from ..encoded_array import EncodedRaggedArray, as_encoded_array
from ..ragged import LazyRaggedArray
from ..rows import RowView


def _device():
    dev = config.default_device()
    if dev.type != "cuda":
        raise nv.NativeLibraryError("pileups need a CUDA device: bionumpy_b200 has no CPU fallback")
    return dev


def _int64(values, device):
    return torch.as_tensor(np.asarray(values) if not isinstance(values, torch.Tensor) else values).to(
        device, torch.int64).contiguous()


def _start_stop(intervals, device):
    return _int64(intervals.start, device), _int64(intervals.stop, device)


def coverage_runs(start, stop, size, mode):
    """The runs of the coverage of global intervals [start, stop) on [0, size) (device int64): (run_starts int64[R + 1],
    values int64[R], the first bad interval or None), the run count and the bad interval read in one copy."""
    keys, _, _, status = ops.interval_events(start, stop, size=size)
    keys = torch.sort(keys).values
    starts, values, n_runs = ops.pileup_runs(keys, size, mode)
    n, bad = torch.cat([n_runs, status[nv.ST_BAD_BASE:nv.ST_BAD_BASE + 1]]).cpu().tolist()
    return starts[:n + 1], values[:n], None if bad == nv.INT64_MAX else bad


def _raise_bad(bad, start, stop, size):
    raise ValueError(f"interval {bad} ({int(start[bad])}-{int(stop[bad])}) is not inside [0, {size})")


def get_pileup(intervals, chromosome_size: int) -> "GenomicRunLengthArray":
    """The number of intervals that cover each position of a contig of ``chromosome_size`` (int64 runs).

    >>> intervals = Interval(["chr1", "chr1", "chr1"], [3, 5, 10], [8, 7, 12])
    >>> print(get_pileup(intervals, 20))
    [0 0 0 1 1 2 2 1 0 0 1 1 0 0 0 0 0 0 0 0]

    An interval with start < 0, stop < start or stop > chromosome_size raises ValueError naming the first one."""
    start, stop = _start_stop(intervals, _device())
    size = int(chromosome_size)
    runs, values, bad = coverage_runs(start, stop, size, nv.PILEUP_COUNT)
    if bad is not None:
        _raise_bad(bad, start, stop, size)
    return GenomicRunLengthArray(runs, values, size)


def get_boolean_mask(intervals, chromosome_size: int) -> "GenomicRunLengthArray":
    """Where any interval covers the contig (bool runs); the intervals need not be sorted.  Bounds as get_pileup."""
    start, stop = _start_stop(intervals, _device())
    size = int(chromosome_size)
    runs, values, bad = coverage_runs(start, stop, size, nv.PILEUP_ANY)
    if bad is not None:
        _raise_bad(bad, start, stop, size)
    return GenomicRunLengthArray(runs, values.to(torch.bool), size)


def merge_intervals(intervals, distance: int = 0):
    """Merge sorted intervals (arithmetics/intervals.py:270-304): stops = the running max of stop (+ distance when it
    is positive); a row starts a new interval iff its start is past the previous row's stops, so touching intervals
    merge.  Each merged interval is the first row of its group with the group's largest stop, in the record type
    given.  Rows may hold several chromosomes when each chromosome's rows are consecutive; a merge never crosses a
    change of chromosome name.  A start that decreases inside a chromosome raises AssertionError.  Chromosome names
    given as a NumPy array or tuple of str are moved to the device as text first; a record without a chromosome field
    is one chromosome."""
    if len(intervals) == 0:
        return intervals
    dev = _device()
    start, stop = _start_stop(intervals, dev)
    same = None
    chrom = getattr(intervals, "chromosome", None)
    if isinstance(chrom, (np.ndarray, tuple, list)):
        chrom = as_encoded_array([str(c) for c in chrom])
        intervals = replace(intervals, chromosome=chrom)
    if isinstance(chrom, EncodedRaggedArray):
        rows = RowView(chrom)
        same = ops.rows_equal_prev(rows.base, rows.starts, rows.lens)
    elif chrom is not None:
        raise TypeError(f"merge_intervals: chromosome names must be text, not {type(chrom).__name__}")
    first, stops, n_out, status = ops.interval_merge(start, stop, same, distance)
    k, bad = torch.cat([n_out, status[nv.ST_BAD_BASE:nv.ST_BAD_BASE + 1]]).cpu().tolist()
    if bad != nv.INT64_MAX:
        raise AssertionError("merge_intervals requires intervals sorted on start position")
    return replace(intervals[first[:k]], stop=stops[:k])


def _format(values: np.ndarray) -> str:
    if values.size <= 20:
        return np.array2string(values, max_line_width=10 ** 6)
    head = np.array2string(values[:3], max_line_width=10 ** 6)
    tail = np.array2string(values[-3:], max_line_width=10 ** 6)
    return f"{head[:-1]} ... {tail[1:]}"


class GenomicRunLengthArray:
    """A track on one contig as runs on the device: ``starts``, ``ends`` and ``values`` are CUDA tensors, ``len()`` is
    the contig size.  The runs are non-empty and no two neighbouring runs have the same value; the first starts at 0
    and the last ends at the size.  Values are integers or bool: the run kernels compute in int64."""

    def __init__(self, events, values, size=None):
        if values.is_floating_point() or values.is_complex():
            raise TypeError(f"run-length values must be integers or bool, not {values.dtype}")
        self._events = events            # int64[R + 1]: run starts and the size
        self._values = values
        self._size = None if size is None else int(size)

    @classmethod
    def from_runs(cls, starts, ends, values):
        """Runs given by their starts, ends and values (host or device, canonical; integer or bool values)."""
        dev = _device()
        s, e = _int64(starts, dev), _int64(ends, dev)
        return cls(torch.cat([s, e[-1:]]), torch.as_tensor(np.asarray(values) if not isinstance(values, torch.Tensor)
                                                              else values).to(dev))

    @property
    def starts(self):
        return self._events[:-1]

    @property
    def ends(self):
        return self._events[1:]

    @property
    def values(self):
        return self._values

    @property
    def dtype(self):
        return self._values.dtype

    def __len__(self):
        if self._size is None:
            self._size = int(self._events[-1].item())
        return self._size

    def _values64(self):
        return self._values.to(torch.int64).contiguous()

    def _cast(self, t):
        """int64 kernel output in the track's dtype.  Every value of the track lies in its dtype's range, so clamping
        to that range first changes only the int64 identity of an empty row's max / min, which becomes the dtype's
        lowest / highest value as RaggedArray gives (a plain cast would wrap INT64_MIN to 0 and INT64_MAX to -1)."""
        dtype = self._values.dtype
        if dtype == torch.bool:
            return t != 0
        if dtype != torch.int64:
            info = torch.iinfo(dtype)
            t = t.clamp(info.min, info.max)
        return t.to(dtype)

    def astype(self, dtype):
        """The runs with their values converted to another integer or bool type (a conversion that maps two
        neighbouring values to one value keeps both runs); a floating-point type raises TypeError."""
        dtype = {int: torch.int64, bool: torch.bool, float: torch.float64}.get(dtype, dtype)
        if isinstance(dtype, np.dtype) or (isinstance(dtype, type) and issubclass(dtype, np.generic)):
            dtype = torch.from_numpy(np.zeros(0, dtype=dtype)).dtype
        return GenomicRunLengthArray(self._events, self._values.to(dtype), self._size)

    def to_array(self):
        """The values at every position, a dense CUDA tensor."""
        n = len(self)
        dev = self._events.device
        if n == 0:
            return torch.empty(0, dtype=self._values.dtype, device=dev)
        offsets = torch.tensor([0, n], dtype=torch.int64, device=dev)
        out = ops.runs_extract(self._events, self._values64(), torch.zeros(1, dtype=torch.int64, device=dev),
                               offsets, n)
        return self._cast(out)

    def __array__(self, dtype=None, copy=None):
        a = self.to_array().cpu().numpy()
        return a.astype(dtype) if dtype is not None else a

    def _reduce(self, mode):
        dev = self._events.device
        q0 = torch.zeros(1, dtype=torch.int64, device=dev)
        return ops.runs_reduce(self._events, self._values64(), q0, self._events[-1:].contiguous(), mode)[0]

    def max(self, axis=None, **kwargs):
        return self._cast(self._reduce(nv.RUNS_ANY if self.dtype == torch.bool else nv.RUNS_MAX))

    def min(self, axis=None, **kwargs):
        return self._cast(self._reduce(nv.RUNS_MIN))

    def sum(self, axis=None, **kwargs):
        return self._reduce(nv.RUNS_SUM)

    def mean(self, axis=None, **kwargs):
        return self._reduce(nv.RUNS_SUM).to(torch.float64) / self._events[-1].to(torch.float64)

    def any(self, axis=None, **kwargs):
        return self._reduce(nv.RUNS_ANY) != 0

    def __getitem__(self, idx):
        if isinstance(idx, (int, np.integer)):
            n = len(self)
            i = int(idx) + n if idx < 0 else int(idx)
            if not 0 <= i < n:
                raise IndexError(idx)
            dev = self._events.device
            q = torch.full((1,), i, dtype=torch.int64, device=dev)
            v = ops.runs_extract(self._events, self._values64(), q, torch.tensor([0, 1], device=dev), 1)
            return self._cast(v)[0].item()
        if isinstance(idx, slice):
            return self._slice(idx)
        if hasattr(idx, "start") and hasattr(idx, "stop") and not isinstance(idx, (torch.Tensor, np.ndarray)):
            start, stop = _start_stop(idx, self._events.device)
            return RunsRaggedArray(self, start, stop)
        return self._positions(idx)

    def _positions(self, positions):
        dev = self._events.device
        pos = _int64(positions, dev).reshape(-1)
        n = len(self)
        if pos.numel() and bool(((pos < 0) | (pos >= n)).any().item()):
            raise IndexError(f"positions outside [0, {n})")
        offsets = torch.arange(pos.numel() + 1, dtype=torch.int64, device=dev)
        return self._cast(ops.runs_extract(self._events, self._values64(), pos, offsets, pos.numel()))

    def _slice(self, sl):
        if sl.step not in (None, 1):
            raise NotImplementedError("run-length arrays are sliced with step 1")
        a, b, _ = sl.indices(len(self))
        b = max(a, b)
        runs = self.starts
        bounds = torch.stack([torch.searchsorted(runs, torch.tensor(a, device=runs.device), right=True) - 1,
                              torch.searchsorted(runs, torch.tensor(b, device=runs.device))])
        i0, i1 = bounds.cpu().tolist()
        i1 = max(i1, i0 + 1)
        events = (self._events[i0:i1 + 1] - a).clamp_(0, b - a)
        return GenomicRunLengthArray(events, self._values[i0:i1], b - a)

    def __repr__(self):
        if len(self) <= 20:
            return _format(self.to_array().cpu().numpy())
        return _format(np.concatenate([self[:3].to_array().cpu().numpy(), self[len(self) - 3:].to_array().cpu().numpy()]))

    __str__ = __repr__


class RunsRaggedArray(LazyRaggedArray):
    """``track[intervals]``: one row per interval, the track's values over [start, stop) clipped to [0, len(track)),
    the same rows for the fused reductions and the gathered values (a part of an interval outside the track has no
    values).  ``max``, ``min``, ``sum``, ``mean`` and ``any`` along the rows run fused over the runs (no
    synchronisation, the positions are never written); anything else gathers the values (one synchronisation, for
    their number)."""

    def __init__(self, track, start, stop):
        size = len(track)
        start = start.clamp(0, size)
        stop = torch.maximum(stop.clamp(max=size), start)
        super().__init__(stop - start, 0)
        self._track = track
        self._q_start, self._q_stop = start.contiguous(), stop.contiguous()

    def _compute(self):
        offsets = ops.row_offsets(self._lens)
        out = ops.runs_extract(self._track._events, self._track._values64(), self._q_start, offsets,
                               int(offsets[-1].item()))
        return self._track._cast(out)

    def _reduce(self, mode):
        return ops.runs_reduce(self._track._events, self._track._values64(), self._q_start, self._q_stop, mode)

    def max(self, axis=None, **kwargs):
        if axis not in (-1, 1):
            return super().max(axis, **kwargs)
        return self._track._cast(self._reduce(nv.RUNS_ANY if self.dtype == torch.bool else nv.RUNS_MAX))

    def min(self, axis=None, **kwargs):
        if axis not in (-1, 1):
            return super().min(axis, **kwargs)
        return self._track._cast(self._reduce(nv.RUNS_MIN))

    def sum(self, axis=None, **kwargs):
        if axis not in (-1, 1):
            return super().sum(axis, **kwargs)
        return self._reduce(nv.RUNS_SUM)

    def mean(self, axis=None, **kwargs):
        if axis not in (-1, 1):
            return super().mean(axis, **kwargs)
        return self._reduce(nv.RUNS_SUM).to(torch.float64) / self._lens.to(torch.float64)

    def any(self, axis=None, **kwargs):
        if axis not in (-1, 1):
            return super().any(axis, **kwargs)
        return self._reduce(nv.RUNS_ANY) != 0

    @property
    def dtype(self):
        return self._track.dtype
