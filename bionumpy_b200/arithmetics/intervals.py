"""Pileups, masks and merges of intervals on one contig (mirror of bionumpy/arithmetics/intervals.py:19-304).

  get_pileup / get_boolean_mask : every interval becomes two event keys (bnpk_interval_events), torch.sort orders them
                                  and one look-back pass writes the runs of the coverage (bnpk_pileup_runs); one
                                  synchronisation reads the run count and the first bad interval.
  merge_intervals               : the reference's running-max rule as one segmented look-back scan
                                  (bnpk_interval_merge), segments cut where the chromosome name changes
                                  (bnpk_rows_equal_prev); one synchronisation.
  GenomicRunLengthArray         : runs on the device; indexing by intervals gives a lazy ragged result whose per-row
                                  max / min / sum / mean / any run fused over the runs (bnpk_runs_reduce) and whose
                                  values, when asked for, are gathered by bnpk_runs_extract.
  FloatRunLengthArray           : the same with float64 values: fused reductions by bnpk_track_f64_reduce (sums with
                                  the same bits on every call), operators by bnpk_track_f64_combine, and the gathers and
                                  bedGraph rows of the integer kernels through an int64 view of the values' bits."""
import numpy as np
import torch

from .. import _native as nv
from .. import config, ops
from ..datatypes import replace
from ..encoded_array import BaseEncoding, EncodedArray, EncodedRaggedArray, as_encoded_array
from ..ragged import LazyRaggedArray
from ..rows import RowView


def _device():
    dev = config.default_device()
    if dev.type != "cuda":
        raise nv.NativeLibraryError("pileups need a CUDA device: bionumpy_b200 has no CPU fallback")
    return dev


def to_device(array, device):
    """A host NumPy array on the device through pinned memory, without waiting for the copy."""
    return torch.from_numpy(np.array(array, copy=True)).pin_memory().to(device, non_blocking=True)


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
    n, st = ops.read_back(n_runs, status)
    return starts[:n + 1], values[:n], st.fault


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
    k, st = ops.read_back(n_out, status)
    if st.fault is not None:
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

    def _reduce_rows(self, q_start, q_stop, mode):
        """The reduction ``mode`` (nv.RUNS_*) of the track over every query [q_start, q_stop): max and min in the
        track's dtype, the sum as the kernel gives it, any as bool.  The one place the reductions reach a kernel."""
        if mode == nv.RUNS_MAX and self.dtype == torch.bool:
            mode = nv.RUNS_ANY                  # the largest of bool values
        out = ops.runs_reduce(self._events, self._values64(), q_start, q_stop, mode)
        if mode == nv.RUNS_ANY:
            return out != 0
        return self._cast(out) if mode != nv.RUNS_SUM else out

    def _reduce(self, mode):
        dev = self._events.device
        q0 = torch.zeros(1, dtype=torch.int64, device=dev)
        return self._reduce_rows(q0, self._events[-1:].contiguous(), mode)[0]

    def max(self, axis=None, **kwargs):
        return self._reduce(nv.RUNS_MAX)

    def min(self, axis=None, **kwargs):
        return self._reduce(nv.RUNS_MIN)

    def sum(self, axis=None, **kwargs):
        return self._reduce(nv.RUNS_SUM)

    def mean(self, axis=None, **kwargs):
        return self._reduce(nv.RUNS_SUM).to(torch.float64) / self._events[-1].to(torch.float64)

    def any(self, axis=None, **kwargs):
        return self._reduce(nv.RUNS_ANY)

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
        return type(self)(events, self._values[i0:i1], b - a)

    def to_bedgraph(self, sequence_name):
        """The runs as BedGraph rows on contig ``sequence_name`` (arithmetics/intervals.py:119-121): every run as it
        is stored, the value in the track's dtype (bool as 0 / 1 when written, where the reference writes True /
        False).  The chromosome column is the name's bytes, viewed by every row; one synchronisation."""
        from ..datatypes import BedGraph
        dev = self._events.device
        n = len(self)
        if n == 0:
            empty = torch.zeros(0, dtype=torch.int64, device=dev)
            no_names = EncodedRaggedArray(EncodedArray(torch.zeros(0, dtype=torch.uint8, device=dev), BaseEncoding),
                                          torch.zeros(0, dtype=torch.int32, device=dev))
            return BedGraph(no_names, empty, empty, self._values[:0])
        ends = torch.tensor([0, n], dtype=torch.int64, device=dev)
        _, start, stop, value, n_out = ops.runs_to_intervals(self._events, self._values64(), ends, nv.RUNS_TO_ALL)
        k = int(n_out.cpu()[0])
        name = torch.frombuffer(bytearray(str(sequence_name).encode()), dtype=torch.uint8).to(dev)
        chrom = EncodedRaggedArray(EncodedArray(name, BaseEncoding), torch.full((k,), name.numel(), dtype=torch.int32,
                                                                                 device=dev),
                                   starts=torch.zeros(k, dtype=torch.int64, device=dev))
        return BedGraph(chrom, start[:k], stop[:k], self._cast(value[:k]))

    def __repr__(self):
        if len(self) <= 20:
            return _format(self.to_array().cpu().numpy())
        return _format(np.concatenate([self[:3].to_array().cpu().numpy(), self[len(self) - 3:].to_array().cpu().numpy()]))

    __str__ = __repr__

    def __array_ufunc__(self, ufunc, method, *inputs, **kwargs):
        """The ufuncs of TRACK_UFUNCS between tracks of one size and integer or bool scalars run on the runs
        (bnpk_runs_combine, one synchronisation); any other call gets the dense arrays."""
        out = track_ufunc(ufunc, method, inputs, kwargs)
        if out is not None:
            return out
        return getattr(ufunc, method)(*[np.asarray(x) if isinstance(x, GenomicRunLengthArray) else x
                                        for x in inputs], **kwargs)


def _binary(ufunc):
    return (lambda self, other: ufunc(self, other)), (lambda self, other: ufunc(other, self))


def _add_operators(cls):
    """The Python operators of a track class as the ufuncs its __array_ufunc__ serves."""
    for name, ufunc in (("and", np.bitwise_and), ("or", np.bitwise_or), ("xor", np.bitwise_xor), ("add", np.add),
                        ("sub", np.subtract), ("mul", np.multiply)):
        forward, reflected = _binary(ufunc)
        setattr(cls, f"__{name}__", forward)
        setattr(cls, f"__r{name}__", reflected)
    for name, ufunc in (("eq", np.equal), ("ne", np.not_equal), ("lt", np.less), ("le", np.less_equal),
                        ("gt", np.greater), ("ge", np.greater_equal)):
        setattr(cls, f"__{name}__", _binary(ufunc)[0])
    cls.__invert__ = lambda self: np.invert(self)
    cls.__neg__ = lambda self: np.negative(self)
    cls.__hash__ = None
    return cls


_add_operators(GenomicRunLengthArray)


class FloatRunLengthArray(GenomicRunLengthArray):
    """A track of float64 runs.  float16 and float32 values (and integer ones) are converted to float64; neighbouring
    runs are one run only when their values are bitwise equal, so -0.0 next to +0.0 stays two runs and NaN runs are
    never merged with a different NaN.  max / min / sum / mean / any follow NumPy: a NaN in a range makes max, min, sum
    and mean NaN, any counts it as true, and an empty range gives -inf, +inf, 0.0, NaN and False.  Sums are rounded
    per run and added in a fixed order: the same bits on every call."""

    def __init__(self, events, values, size=None):
        if values.is_complex():
            raise TypeError(f"run-length values must be real, not {values.dtype}")
        self._events = events
        self._values = values.to(torch.float64)
        self._size = None if size is None else int(size)

    def _values64(self):
        return self._values.contiguous().view(torch.int64)

    def _cast(self, t):
        return t.view(torch.float64)

    def astype(self, dtype):
        raise TypeError("float tracks are not converted to another type")

    def _reduce_rows(self, q_start, q_stop, mode):
        out = ops.track_f64_reduce(self._events, self._values.contiguous(), q_start, q_stop, mode)
        return out != 0 if mode == nv.RUNS_ANY else out


def _is_float_track(x):
    return isinstance(getattr(x, "_global", x), FloatRunLengthArray)


def _truediv(self, other):
    return np.true_divide(self, other) if _is_float_track(self) or _is_float_track(other) else NotImplemented


def _rtruediv(self, other):
    return np.true_divide(other, self) if _is_float_track(self) or _is_float_track(other) else NotImplemented


GenomicRunLengthArray.__truediv__ = _truediv
GenomicRunLengthArray.__rtruediv__ = _rtruediv

# ufunc -> the kernel's operator; the logical ones first map each value to (value != 0)
TRACK_UFUNCS = {np.add: nv.OP_ADD, np.subtract: nv.OP_SUB, np.multiply: nv.OP_MUL, np.bitwise_and: nv.OP_AND,
                np.bitwise_or: nv.OP_OR, np.bitwise_xor: nv.OP_XOR, np.minimum: nv.OP_MIN, np.maximum: nv.OP_MAX,
                np.equal: nv.OP_EQ, np.not_equal: nv.OP_NE, np.less: nv.OP_LT, np.less_equal: nv.OP_LE,
                np.greater: nv.OP_GT, np.greater_equal: nv.OP_GE, np.logical_and: nv.OP_AND,
                np.logical_or: nv.OP_OR, np.logical_xor: nv.OP_XOR}
_LOGICAL = (np.logical_and, np.logical_or, np.logical_xor)


def _is_int_scalar(x):
    return isinstance(x, (bool, int, np.bool_, np.integer))


def _probe(x):
    """What NumPy's type rules see of an operand: a one-element array of the track's computed dtype (bool, or int64 for
    every integer track), or the scalar itself."""
    if isinstance(x, GenomicRunLengthArray):
        return np.zeros(1, dtype=np.bool_ if x.dtype == torch.bool else np.int64)
    return x


def track_ufunc(ufunc, method, inputs, kwargs):
    """``ufunc(*inputs)`` on run-length tracks, or None when the call is not one the runs serve (another ufunc or
    method, keyword arguments, a float or non-scalar operand).  Unary ufuncs are binary ones with a scalar: ~x is
    x ^ -1 (x ^ True for bool), -x is 0 - x and logical_not(x) is x == 0.  The result dtype is NumPy's on the dense
    arrays, except that integer tracks narrower than int64 are computed, and returned, as int64; a result NumPy gives
    as float or as an unsigned type wider than uint8 takes the dense path (None).  Tracks of different
    sizes raise ValueError; what NumPy refuses (bool - bool, -bool) raises its TypeError."""
    if method != "__call__" or kwargs:
        return None
    if any(isinstance(x, FloatRunLengthArray) for x in inputs):
        return float_track_ufunc(ufunc, inputs)
    if len(inputs) == 1:
        (x,) = inputs
        if not isinstance(x, GenomicRunLengthArray):
            return None
        if ufunc is np.invert:
            np.invert(_probe(x))
            return track_ufunc(np.bitwise_xor, method, (x, True if x.dtype == torch.bool else -1), kwargs)
        if ufunc is np.negative:
            np.negative(_probe(x))
            return track_ufunc(np.subtract, method, (0, x), kwargs)
        if ufunc is np.logical_not:
            return track_ufunc(np.equal, method, (x, False if x.dtype == torch.bool else 0), kwargs)
        return None
    if len(inputs) != 2 or ufunc not in TRACK_UFUNCS:
        return None
    if not all(isinstance(x, GenomicRunLengthArray) or _is_int_scalar(x) for x in inputs):
        return None
    tracks = [x for x in inputs if isinstance(x, GenomicRunLengthArray)]
    size = len(tracks[0])
    if any(len(t) != size for t in tracks):
        raise ValueError(f"tracks of sizes {len(tracks[0])} and {len(tracks[1])} cannot be combined")
    dtype = ufunc(*[_probe(x) for x in inputs]).dtype
    if dtype.kind not in "biu" or (dtype.kind == "u" and dtype.itemsize > 1):
        return None              # float, and uint16 / 32 / 64 (a bool track with such a scalar): the dense path
    dev = tracks[0]._events.device
    if ufunc not in _LOGICAL and any(_is_int_scalar(x) and not -2 ** 63 <= int(x) < 2 ** 63 for x in inputs):
        if dtype != np.bool_:
            return None
        # a comparison with an integer that no int64 equals has one result at every position, NumPy's
        value = torch.full((1,), bool(ufunc(*[_probe(x) for x in inputs])[0]), dtype=torch.bool, device=dev)
        return GenomicRunLengthArray(torch.arange(2, dtype=torch.int64, device=dev) * size, value, size)
    op = TRACK_UFUNCS[ufunc]
    if dtype == np.bool_ and ufunc in (np.add, np.multiply):
        op = nv.OP_OR if ufunc is np.add else nv.OP_AND          # NumPy's bool + and *
    runs = []
    for x in inputs:
        if isinstance(x, GenomicRunLengthArray):
            values = x._values64() if ufunc not in _LOGICAL or x.dtype == torch.bool else (x._values != 0).to(torch.int64)
            runs.append((x._events, values))
        else:
            v = int(bool(x)) if ufunc in _LOGICAL else int(x)
            runs.append((torch.arange(2, dtype=torch.int64, device=dev) * size,      # made on the device: no copy
                         torch.full((1,), v, dtype=torch.int64, device=dev)))
    (a_starts, a_values), (b_starts, b_values) = runs
    if size == 0:          # a size-0 track has one empty run; the kernel needs both sides alike
        a_starts, a_values = a_starts[:1], a_values[:0]
        b_starts, b_values = b_starts[:1], b_values[:0]
    starts, values, n_runs = ops.runs_combine(a_starts.contiguous(), a_values.contiguous(), b_starts.contiguous(),
                                              b_values.contiguous(), op)
    n = int(n_runs.item())
    if size == 0:
        starts, values, n = torch.zeros(2, dtype=torch.int64, device=dev), torch.zeros(1, dtype=torch.int64, device=dev), 1
    if dtype == np.bool_:
        values = values[:n] != 0
    elif dtype.itemsize < 8:
        # only a bool track with a narrower NumPy integer scalar gets here (True + np.int8(127)): NumPy's dtype, and
        # the int64 result wrapped into it as NumPy wraps; the two values of such a track stay distinct
        values = values[:n].to(torch.from_numpy(np.zeros(0, dtype=dtype)).dtype)
    else:
        values = values[:n]
    return GenomicRunLengthArray(starts[:n + 1], values, size)


FLOAT_UFUNCS = {np.add: nv.OP_ADD, np.subtract: nv.OP_SUB, np.multiply: nv.OP_MUL, np.true_divide: nv.OP_DIV,
                np.minimum: nv.OP_MIN, np.maximum: nv.OP_MAX, np.equal: nv.OP_EQ, np.not_equal: nv.OP_NE,
                np.less: nv.OP_LT, np.less_equal: nv.OP_LE, np.greater: nv.OP_GT, np.greater_equal: nv.OP_GE}
_COMPARISONS = (np.equal, np.not_equal, np.less, np.less_equal, np.greater, np.greater_equal)


def float_track_ufunc(ufunc, inputs):
    """``ufunc(*inputs)`` where an operand is a FloatRunLengthArray, or None for a call the runs do not serve.  The
    other operand is a float track, an integer or bool track (its values converted to float64 as NumPy converts them)
    or an int or float scalar.  np.negative flips the sign bit, np.logical_not(x) is x == 0; FLOAT_UFUNCS run on the
    runs (bnpk_track_f64_combine, one synchronisation): comparisons give bool tracks, the others float tracks.  Tracks
    of different sizes raise ValueError."""
    if len(inputs) == 1:
        (x,) = inputs
        if ufunc is np.negative:
            flipped = x._values.contiguous().view(torch.int64) ^ torch.iinfo(torch.int64).min
            return FloatRunLengthArray(x._events, flipped.view(torch.float64), x._size)
        if ufunc is np.logical_not:
            return float_track_ufunc(np.equal, (x, 0.0))
        return None
    if len(inputs) != 2 or ufunc not in FLOAT_UFUNCS:
        return None
    scalar = (bool, int, float, np.bool_, np.integer, np.floating)
    if not all(isinstance(x, GenomicRunLengthArray) or isinstance(x, scalar) for x in inputs):
        return None
    if any(isinstance(x, (int, np.integer)) and abs(int(x)) >= 2 ** 1024 for x in inputs):
        return None
    tracks = [x for x in inputs if isinstance(x, GenomicRunLengthArray)]
    size = len(tracks[0])
    if any(len(t) != size for t in tracks):
        raise ValueError(f"tracks of sizes {len(tracks[0])} and {len(tracks[1])} cannot be combined")
    dev = tracks[0]._events.device
    runs = []
    for x in inputs:
        if isinstance(x, GenomicRunLengthArray):
            runs.append((x._events, x._values.to(torch.float64)))
        else:
            runs.append((torch.arange(2, dtype=torch.int64, device=dev) * size,      # made on the device: no copy
                         torch.full((1,), float(x), dtype=torch.float64, device=dev)))
    (a_starts, a_values), (b_starts, b_values) = runs
    if size == 0:          # a size-0 track has one empty run; the kernel needs both sides alike
        a_starts, a_values = a_starts[:1], a_values[:0]
        b_starts, b_values = b_starts[:1], b_values[:0]
    starts, values, n_runs = ops.track_f64_combine(a_starts.contiguous(), a_values.contiguous(),
                                                   b_starts.contiguous(), b_values.contiguous(), FLOAT_UFUNCS[ufunc])
    n = int(n_runs.item())
    if size == 0:
        starts, values, n = torch.zeros(2, dtype=torch.int64, device=dev), torch.zeros(1, dtype=torch.float64,
                                                                                      device=dev), 1
    if ufunc in _COMPARISONS:
        return GenomicRunLengthArray(starts[:n + 1], values[:n] != 0, size)
    return FloatRunLengthArray(starts[:n + 1], values[:n], size)


class RunsRaggedArray(LazyRaggedArray):
    """``track[intervals]``: one row per interval, the track's values over [start, stop) clipped to [0, len(track)),
    the same rows for the fused reductions and the gathered values (a part of an interval outside the track has no
    values).  ``max``, ``min``, ``sum``, ``mean`` and ``any`` along the rows run fused over the runs (no
    synchronisation, the positions are never written); anything else gathers the values (one synchronisation, for
    their number).  ``reverse`` (a bool or uint8 device tensor, one flag per row, or None) gives the values of the
    flagged rows back to front, as the windows of '-' strand features are read (an index permutation after the gather,
    which at its peak needs about three times the gather's memory); the reductions along the rows do not depend on
    it.  ``sum(axis=0)`` and ``mean(axis=0)`` of rows of one length run fused over the runs too
    (bnpk_runs_column_sum / bnpk_track_f64_column_sum): one synchronisation, for the width and the length check."""

    def __init__(self, track, start, stop, reverse=None):
        size = len(track)
        start = start.clamp(0, size)
        stop = torch.maximum(stop.clamp(max=size), start)
        super().__init__(stop - start, 0)
        self._track = track
        self._q_start, self._q_stop = start.contiguous(), stop.contiguous()
        self._reverse = None if reverse is None else reverse.to(torch.uint8).contiguous()

    def _compute(self):
        offsets = ops.row_offsets(self._lens)
        total = int(offsets[-1].item())
        out = ops.runs_extract(self._track._events, self._track._values64(), self._q_start, offsets, total)
        if self._reverse is not None and total:
            # the value at flat index j of a reversed row [o, o + L) is the gathered one at 2o + L - 1 - j: one mirror
            # point per row (-1 on forward rows) spread over the row's positions, the permutation built in place.  At
            # its peak this holds two int64 and one bool per position beside the gathered values: about three times
            # the memory of an unstranded gather.
            lens = self._lens.to(torch.int64)
            mirror = torch.where(self._reverse != 0, 2 * offsets[:-1] + lens - 1, -1)
            src = torch.repeat_interleave(mirror, lens, output_size=total)
            idx = torch.arange(total, dtype=torch.int64, device=lens.device)
            flip = src >= 0
            torch.where(flip, src.sub_(idx), idx, out=idx)
            del src, flip
            out = out[idx]
        return self._track._cast(out)

    def _reduce(self, mode):
        return self._track._reduce_rows(self._q_start, self._q_stop, mode)

    def _column_sum(self):
        """The sum of every column of rows of one length, and the row count: int64 for integer and bool tracks,
        float64 for float tracks.  One synchronisation reads the width and the number of rows of another length."""
        n = len(self)
        lens = self._lens.to(torch.int64)
        if n == 0:
            raise NotImplementedError("mean(axis=0) needs rows of one length: there are no rows")
        width, n_other = ops.read_back(lens[:1], (lens != lens[0]).sum())
        if n_other:
            raise NotImplementedError(f"mean(axis=0) needs rows of one length: {n_other} of the {n} rows differ in "
                                      f"length from the first ({width})")
        track = self._track
        if isinstance(track, FloatRunLengthArray):
            return ops.track_f64_column_sum(track._events, track._values.contiguous(), self._q_start, width,
                                            self._reverse), n
        return ops.runs_column_sum(track._events, track._values64(), self._q_start, width, self._reverse), n

    def max(self, axis=None, **kwargs):
        if axis not in (-1, 1):
            return super().max(axis, **kwargs)
        return self._reduce(nv.RUNS_MAX)

    def min(self, axis=None, **kwargs):
        if axis not in (-1, 1):
            return super().min(axis, **kwargs)
        return self._reduce(nv.RUNS_MIN)

    def sum(self, axis=None, **kwargs):
        if axis == 0:
            return self._column_sum()[0]
        if axis not in (-1, 1):
            return super().sum(axis, **kwargs)
        return self._reduce(nv.RUNS_SUM)

    def mean(self, axis=None, **kwargs):
        if axis == 0:
            total, n = self._column_sum()
            # a true division: torch divides by a Python scalar as a multiply by its reciprocal
            return total.to(torch.float64) / torch.full_like(total, n, dtype=torch.float64)
        if axis not in (-1, 1):
            return super().mean(axis, **kwargs)
        return self._reduce(nv.RUNS_SUM).to(torch.float64) / self._lens.to(torch.float64)

    def any(self, axis=None, **kwargs):
        if axis not in (-1, 1):
            return super().any(axis, **kwargs)
        return self._reduce(nv.RUNS_ANY)

    @property
    def dtype(self):
        return self._track.dtype


# --------------------------------------------------------------------------------------------------------------------
# interval sets (arithmetics/intervals.py:235-342)
# --------------------------------------------------------------------------------------------------------------------
NAME_SLOTS, NAME_BYTES = 4096, 1 << 16      # the distinct-name runs read back in the one synchronisation


def _text_column(intervals):
    chrom = intervals.chromosome
    if isinstance(chrom, (np.ndarray, tuple, list)):
        chrom = as_encoded_array([str(c) for c in chrom])
    if not isinstance(chrom, EncodedRaggedArray):
        raise TypeError(f"chromosome names must be text, not {type(chrom).__name__}")
    return chrom


def _name_runs(rows, slots=NAME_SLOTS, nbytes=NAME_BYTES):
    """The first ``slots`` rows that start a run of equal names, packed for the host: [count, bytes] as int64, each
    slot's length as int64 and the slots' bytes end to end (``nbytes``), all uint8; no synchronisation."""
    dev, n = rows.base.device, rows.lens.numel()
    first = ops.rows_equal_prev(rows.base, rows.starts, rows.lens) == 0
    pos = torch.cumsum(first, 0) - 1
    slot = torch.where(first & (pos < slots), pos, torch.full_like(pos, slots))
    row = torch.zeros(slots + 1, dtype=torch.int64, device=dev).scatter_(
        0, slot, torch.arange(n, dtype=torch.int64, device=dev))[:slots]
    count = first.sum().reshape(1)
    total = torch.where(first, rows.lens.to(torch.int64), 0).sum().reshape(1)       # of every run, not only the slots'
    lens = torch.where(torch.arange(slots, device=dev) < count, rows.lens[row].to(torch.int64), 0)
    ends = torch.cumsum(lens, 0)
    j = torch.arange(nbytes, dtype=torch.int64, device=dev)
    r = torch.searchsorted(ends, j, right=True).clamp_(max=slots - 1)
    src = (rows.starts[row[r]] + j - (ends[r] - lens[r])).clamp_(0, max(rows.base.numel() - 1, 0))
    data = torch.where(j < ends[-1], rows.base[src], 0).to(torch.uint8)
    return torch.cat([torch.cat([count, total, lens]).view(torch.uint8), data])


def _unpack_names(packed, rows):
    """The distinct names of _name_runs' packing; more runs or bytes than it holds are read again, exactly (one more
    synchronisation)."""
    count, total = np.frombuffer(packed[:16].tobytes(), dtype=np.int64).tolist()
    slots = NAME_SLOTS
    if count > NAME_SLOTS or total > NAME_BYTES:
        slots = count
        packed = _name_runs(rows, count, total).cpu().numpy()
    lens = np.frombuffer(packed[16:16 + 8 * count].tobytes(), dtype=np.int64).tolist()
    data = packed[16 + 8 * slots:].tobytes()
    ends = np.cumsum(lens).tolist()
    return {data[e - n:e].decode() for e, n in zip(ends, lens)}


def chromosome_ranks(columns, key=None, sort_order=None):
    """The rank of every row's chromosome name in each text column (int64 device tensors), in one synchronisation:
    the rows that start a run of equal names (bnpk_rows_equal_prev) are the only names copied to the host, where the
    distinct names are ranked by ``key(name)`` (equal keys share a rank), by their position in ``sort_order`` (a name
    missing from it raises KeyError) or, by default, as bytes; a byte-sorted table of them maps every row to its rank on
    the device (bnpk_name_lookup)."""
    views = [RowView(c) for c in columns]
    live = [v for v in views if v.lens.numel()]
    if not live:
        return [torch.zeros(0, dtype=torch.int64, device=v.base.device) for v in views]
    packed = torch.cat([_name_runs(v) for v in live]).cpu().numpy()
    size = packed.size // len(live)
    names = set()
    for i, v in enumerate(live):
        names |= _unpack_names(packed[i * size:(i + 1) * size], v)
    if sort_order is not None:
        order = {name: i for i, name in enumerate(sort_order)}
        missing = sorted(names - set(order))
        if missing:
            raise KeyError(missing[0])
        rank = {n: order[n] for n in names}
    else:
        key = key or (lambda n: n.encode())
        keys = {n: key(n) for n in names}
        rank, r, prev = {}, -1, object()
        for n in sorted(names, key=keys.__getitem__):
            if r < 0 or keys[n] != prev:
                r, prev = r + 1, keys[n]
            rank[n] = r
    table = sorted(names, key=str.encode)
    raw = [n.encode() for n in table]
    dev = views[0].base.device
    text = to_device(np.frombuffer(b"".join(raw) or b"\0", dtype=np.uint8), dev)
    offsets = to_device(np.cumsum([0] + [len(b) for b in raw]).astype(np.int64), dev)
    of_table = to_device(np.array([rank[n] for n in table], dtype=np.int64), dev)
    out = []
    for v in views:
        if v.lens.numel() == 0:
            out.append(torch.zeros(0, dtype=torch.int64, device=dev))
            continue
        ids, _ = ops.name_lookup(v.base, v.starts, v.lens, text, offsets)
        out.append(of_table[ids.to(torch.int64)])
    return out


def lexsort_order(*keys):
    """np.lexsort(keys) (the last key is the primary one) as stable torch.sort passes on the device."""
    order = torch.sort(keys[0], stable=True).indices
    for k in keys[1:]:
        order = order[torch.sort(k[order], stable=True).indices]
    return order


def sort_intervals(intervals, chromosome_key_function=lambda x: x, sort_order=None):
    """Intervals ordered by (chromosome_key_function(chromosome), start, stop), stably (arithmetics/intervals.py:
    235-256); with ``sort_order`` the chromosomes come in that order and a chromosome missing from it raises KeyError.
    One synchronisation, for the distinct chromosome names."""
    if len(intervals) == 0:
        return intervals
    dev = _device()
    start, stop = _start_stop(intervals, dev)
    (rank,) = chromosome_ranks([_text_column(intervals)], chromosome_key_function, sort_order)
    return intervals[lexsort_order(stop, start, rank)]


def _sweep(a, b, start, stop, same=None):
    """Rows of concatenate(a, b) ordered by ``start`` (the device order over the concatenated rows) paired with
    ``stop`` by bnpk_interval_intersect: the emitted rows with their stops replaced, one synchronisation."""
    from ..datatypes import concatenate
    rows, stops, n_out, _ = ops.interval_intersect(start[0], stop, same)
    both, (k,) = concatenate(a, b, extra=[n_out])
    return replace(both[start[1][rows[:k]]], stop=stops[:k])


def intersect(intervals_a, intervals_b):
    """The reference's sorted sweep (arithmetics/intervals.py:317-325), which ignores the chromosome: the rows of both
    sets ordered by start (stably), every row whose start lies before the previous sorted stop, with that stop.  Both
    sets must be records of one type.  One synchronisation."""
    dev = _device()
    sa, ea = _start_stop(intervals_a, dev)
    sb, eb = _start_stop(intervals_b, dev)
    start, stop = torch.cat([sa, sb]), torch.cat([ea, eb])
    order = torch.sort(start, stable=True).indices
    return _sweep(intervals_a, intervals_b, (start[order], order), torch.sort(stop).values)


def global_intersect(intervals_b, intervals_a):
    """intersect on every chromosome (arithmetics/intervals.py:328-335, argument order kept: the rows of intervals_a
    come first): rows ordered by (chromosome name as bytes, start), stably, stops by (name, stop).  Unlike the
    reference, the last stop of one chromosome is never compared with the first start of the next, so a = chr1:100-200
    and b = chr2:10-20 intersect to nothing (the reference gives chr2:10-200).  Two synchronisations."""
    dev = _device()
    sa, ea = _start_stop(intervals_a, dev)
    sb, eb = _start_stop(intervals_b, dev)
    ra, rb = chromosome_ranks([_text_column(intervals_a), _text_column(intervals_b)])
    start, stop, rank = torch.cat([sa, sb]), torch.cat([ea, eb]), torch.cat([ra, rb])
    order = lexsort_order(start, rank)
    stops = stop[lexsort_order(stop, rank)]
    r = rank[order]
    same = torch.cat([torch.zeros(1, dtype=torch.bool, device=dev), r[1:] == r[:-1]]).to(torch.uint8)
    return _sweep(intervals_a, intervals_b, (start[order], order), stops, same)


def count_overlap(intervals_a, intervals_b) -> int:
    """The sum over the sorted sweep of both sets of max(previous stop - start, 0) (arithmetics/intervals.py:307-314),
    on one contig: one kernel launch that writes no rows, one synchronisation."""
    dev = _device()
    sa, ea = _start_stop(intervals_a, dev)
    sb, eb = _start_stop(intervals_b, dev)
    start = torch.sort(torch.cat([sa, sb])).values
    stop = torch.sort(torch.cat([ea, eb])).values
    _, _, _, overlap = ops.interval_intersect(start, stop, rows=False)
    return int(overlap.item())


def unique_intersect(intervals_a, intervals_b, genome_size):
    """The rows of intervals_a that overlap any interval of intervals_b (arithmetics/intervals.py:338-342): the mask of
    b, then the fused any() of a's rows over it.  Two synchronisations."""
    mask = get_boolean_mask(intervals_b, genome_size)
    rows = torch.nonzero(mask[intervals_a].any(axis=-1)).reshape(-1)      # one read, then every field by index
    return intervals_a[rows]
