"""Ragged storage on the device: a flat torch tensor plus a row-offset vector.

Stands in for ``npstructures.RaggedArray`` / ``RaggedView2`` (the reference's storage for
``EncodedRaggedArray``, bionumpy/encoded_array.py:161-166, bionumpy/io/file_buffers.py:335-338).
A ragged array is ALWAYS a view ``(base, starts[R], lens[R])``; it is *contiguous* when the rows
tile ``base`` back to back.  Row/column slicing returns new views and moves no data; ``ravel()``
gathers only when the view is not contiguous.
"""
import numpy as np
import torch


def _as_index_tensor(x, device, dtype=torch.int64):
    if isinstance(x, torch.Tensor):
        return x.to(device=device, dtype=dtype)
    return torch.as_tensor(np.asarray(x), dtype=dtype, device=device)


def segment_max(values, rows, n_rows):
    """out[r] = max of values[i] with rows[i] == r, NaN if one of them is NaN; the dtype's lowest value (-inf for
    floats, False for bool: the max of bools is any) where there is none."""
    if values.dtype == torch.bool:
        return segment_sum(values, rows, n_rows) > 0
    low = -float("inf") if values.is_floating_point() else torch.iinfo(values.dtype).min
    out = torch.full((n_rows,), low, dtype=values.dtype, device=values.device)
    out.scatter_reduce_(0, rows, values, "amax", include_self=True)
    if values.is_floating_point():
        nan = torch.zeros(n_rows, dtype=torch.int32, device=values.device)
        nan.index_add_(0, rows, torch.isnan(values).to(torch.int32))
        out = torch.where(nan > 0, torch.full_like(out, float("nan")), out)
    return out


def segment_min(values, rows, n_rows):
    """out[r] = min of values[i] with rows[i] == r, NaN if one of them is NaN; the dtype's highest value (+inf for
    floats, True for bool: the min of bools is all) where there is none."""
    if values.dtype == torch.bool:
        return segment_sum(~values, rows, n_rows) == 0
    return -segment_max(-values, rows, n_rows) if values.is_floating_point() else \
        _segment_min_int(values, rows, n_rows)


def _segment_min_int(values, rows, n_rows):
    out = torch.full((n_rows,), torch.iinfo(values.dtype).max, dtype=values.dtype, device=values.device)
    return out.scatter_reduce_(0, rows, values, "amin", include_self=True)


def segment_sum(values, rows, n_rows):
    """out[r] = the sum of values[i] with rows[i] == r, int64."""
    out = torch.zeros(n_rows, dtype=torch.int64, device=values.device)
    return out.index_add_(0, rows, values.to(torch.int64))


class RaggedShape:
    """(starts, lens) of the rows.  Compared by lengths only, like npstructures.RaggedShape."""

    def __init__(self, lens, starts=None):
        self.lens = lens
        self.starts = starts

    @property
    def lengths(self):
        return self.lens

    def __eq__(self, other):
        o = other.lens if isinstance(other, RaggedShape) else other
        a = self.lens.cpu().numpy().astype(np.int64)
        b = o.cpu().numpy().astype(np.int64) if isinstance(o, torch.Tensor) else np.asarray(o, dtype=np.int64)
        return a.shape == b.shape and bool(np.all(a == b))

    def __repr__(self):
        return f"RaggedShape({self.lens.cpu().tolist()})"


class RaggedArray:
    def __init__(self, data, shape=None, starts=None, contiguous=None):
        """``data``: flat torch tensor (or nested list).  ``shape``: row lengths (list / tensor /
        RaggedShape).  ``starts``: optional row starts into ``data`` (a view)."""
        if shape is None and not isinstance(data, torch.Tensor):
            rows = [np.asarray(r) for r in data]
            shape = [len(r) for r in rows]
            flat = np.concatenate(rows) if rows else np.zeros(0)
            data = torch.as_tensor(flat)
        if isinstance(shape, RaggedShape):
            starts = shape.starts if starts is None else starts
            shape = shape.lens
        if not isinstance(data, torch.Tensor):
            data = torch.as_tensor(np.asarray(data))
        self._data = data
        self._lens = _as_index_tensor(shape, data.device, torch.int32)
        if starts is None:
            ends = torch.cumsum(self._lens.to(torch.int64), 0)
            self._starts = ends - self._lens
            self._contiguous = True
        else:
            self._starts = _as_index_tensor(starts, data.device, torch.int64)
            self._contiguous = bool(contiguous) if contiguous is not None else False

    # -- structure ---------------------------------------------------------------------------
    @property
    def lengths(self):
        return self._lens

    @property
    def _shape(self):
        return RaggedShape(self._lens, self._starts)

    @property
    def shape(self):
        return (len(self), self._lens)

    @property
    def size(self):
        return int(self._lens.sum().item())

    @property
    def dtype(self):
        return self._data.dtype

    @property
    def device(self):
        return self._data.device

    def __len__(self):
        return self._lens.numel()

    def is_contiguous(self):
        return self._contiguous and (len(self) == 0 or (int(self._starts[0].item()) == 0 and self.size == self._data.numel()))

    def ravel(self):
        if self.is_contiguous():
            return self._data
        lens64 = self._lens.to(torch.int64)
        total = int(lens64.sum().item())
        if total == 0:
            return self._data[:0]
        offsets = torch.cumsum(lens64, 0) - lens64
        idx = torch.repeat_interleave(self._starts - offsets, lens64) + torch.arange(total, device=self._data.device)
        return self._data[idx]

    def _view(self, data, lens, starts):
        return self.__class__(data, lens, starts=starts)

    # -- indexing ----------------------------------------------------------------------------
    def _col_slice(self, sl):
        if sl.step not in (None, 1):
            raise NotImplementedError("column step")
        L = self._lens.to(torch.int64)

        def bound(v, default):
            if v is None:
                return default
            if v < 0:
                return torch.clamp(L + v, min=0)
            return torch.clamp(torch.full_like(L, v), max=L)

        a = bound(sl.start, torch.zeros_like(L))
        b = bound(sl.stop, L)
        new_lens = torch.clamp(b - a, min=0).to(torch.int32)
        return self._view(self._data, new_lens, self._starts + a)

    def _row(self, i):
        n = len(self)
        if i < 0:
            i += n
        if not 0 <= i < n:
            raise IndexError(i)
        s = int(self._starts[i].item())
        return self._data[s:s + int(self._lens[i].item())]

    def __getitem__(self, idx):
        if isinstance(idx, tuple):
            if len(idx) != 2:
                raise IndexError("ragged arrays are two-dimensional")
            rows, cols = idx
            if rows is Ellipsis:
                rows = slice(None)
            if isinstance(rows, (int, np.integer)):
                r = self._row(int(rows))
                return r[cols]
            sub = self[rows]
            if isinstance(cols, slice):
                return sub._col_slice(cols)
            if isinstance(cols, (int, np.integer)):
                c = int(cols)
                L = sub._lens.to(torch.int64)
                pos = sub._starts + (c if c >= 0 else L + c)
                return sub._data[pos]
            raise IndexError(f"unsupported column index {cols!r}")
        if isinstance(idx, (int, np.integer)):
            return self._row(int(idx))
        if idx is Ellipsis:
            return self
        if isinstance(idx, slice):
            return self._view(self._data, self._lens[idx], self._starts[idx])
        if isinstance(idx, (list, np.ndarray)):
            idx = torch.as_tensor(np.asarray(idx), device=self._data.device)
        if isinstance(idx, torch.Tensor):
            idx = idx.to(self._data.device)
            return self._view(self._data, self._lens[idx], self._starts[idx])
        raise IndexError(f"unsupported index {idx!r}")

    def __iter__(self):
        starts = self._starts.cpu().tolist()
        lens = self._lens.cpu().tolist()
        for s, l in zip(starts, lens):
            yield self._data[s:s + l]

    def tolist(self):
        flat = self.ravel().cpu().tolist()
        out, o = [], 0
        for l in self._lens.cpu().tolist():
            out.append(flat[o:o + l])
            o += l
        return out

    def to_numpy_rows(self):
        flat = self.ravel().cpu().numpy()
        out, o = [], 0
        for l in self._lens.cpu().tolist():
            out.append(flat[o:o + l])
            o += l
        return out

    # -- elementwise comparison (README.rst:40-41: ``chunk.sequence == "G"``) ---------------------
    def _compare(self, other, op):
        flat = self.ravel()
        if isinstance(other, RaggedArray):
            other = other.ravel()
        res = op(flat, other)
        return RaggedArray(res, self._lens)

    def __eq__(self, other):
        return self._compare(other, torch.eq)

    def __ne__(self, other):
        return self._compare(other, torch.ne)

    def __lt__(self, other):
        return self._compare(other, torch.lt)

    def __le__(self, other):
        return self._compare(other, torch.le)

    def __gt__(self, other):
        return self._compare(other, torch.gt)

    def __ge__(self, other):
        return self._compare(other, torch.ge)

    __hash__ = None

    def max(self, axis=None, **kwargs):
        """np.max: a NaN makes the maximum NaN.  axis=-1: one value per row; an empty row gives the dtype's lowest
        value (-inf for floats)."""
        flat = self.ravel()
        if axis is None:
            return flat.max()
        if axis in (-1, 1):
            rows = torch.repeat_interleave(torch.arange(len(self), device=flat.device), self._lens.to(torch.int64))
            return segment_max(flat, rows, len(self))
        raise NotImplementedError(axis)

    def min(self, axis=None, **kwargs):
        """np.min, the mirror of ``max``: axis=-1 gives one value per row; an empty row gives the dtype's highest value
        (+inf for floats)."""
        flat = self.ravel()
        if axis is None:
            return flat.min()
        if axis in (-1, 1):
            rows = torch.repeat_interleave(torch.arange(len(self), device=flat.device), self._lens.to(torch.int64))
            return segment_min(flat, rows, len(self))
        raise NotImplementedError(axis)

    def sum(self, axis=None, **kwargs):
        if axis is None:
            return self.ravel().sum()
        if axis in (-1, 1):
            flat = self.ravel()
            lens64 = self._lens.to(torch.int64)
            rows = torch.repeat_interleave(torch.arange(len(self), device=flat.device), lens64)
            out = torch.zeros(len(self), dtype=torch.int64, device=flat.device)
            return out.index_add_(0, rows, flat.to(torch.int64))
        raise NotImplementedError(axis)

    def _row_index(self):
        return torch.repeat_interleave(torch.arange(len(self), device=self._data.device), self._lens.to(torch.int64))

    def any(self, axis=None, **kwargs):
        """np.any: axis=-1 gives one bool per row, False for an empty row."""
        flat = self.ravel()
        if axis is None:
            return (flat != 0).any()
        if axis in (-1, 1):
            return segment_sum(flat != 0, self._row_index(), len(self)) > 0
        raise NotImplementedError(axis)

    def mean(self, axis=None, **kwargs):
        """np.mean in float64: axis=-1 gives one value per row, NaN for an empty row; axis=0 one value per column when
        every row has the same length."""
        flat = self.ravel().to(torch.float64)
        if axis is None:
            return flat.mean()
        if axis == 0:
            n = len(self)
            width = int(self._lens[0].item()) if n else 0
            if n == 0 or bool((self._lens != width).any().item()):
                raise NotImplementedError("mean(axis=0) needs rows of one length")
            return flat.reshape(n, width).mean(0)
        if axis in (-1, 1):
            out = torch.zeros(len(self), dtype=torch.float64, device=flat.device)
            return out.index_add_(0, self._row_index(), flat) / self._lens.to(torch.float64)
        raise NotImplementedError(axis)

    def __array__(self, dtype=None, copy=None):
        # np.sum(ragged) and friends: hand NumPy the flat values
        a = self.ravel().cpu().numpy()
        return a.astype(dtype) if dtype is not None else a

    def __repr__(self):
        rows = self.tolist()
        return f"ragged_array({rows})"


class LazyRaggedArray(RaggedArray):
    """A contiguous RaggedArray with max(lens - shrink, 0) values per row (the windows of rows of ``lens`` bases) whose
    flat data ``_compute()`` makes on first use."""

    def __init__(self, lens, shrink):
        self._lens = torch.clamp(lens - shrink, min=0).to(torch.int32)
        ends = torch.cumsum(self._lens.to(torch.int64), 0)
        self._starts = ends - self._lens
        self._contiguous = True
        self._lazy = None

    def _compute(self):
        raise NotImplementedError

    # RaggedArray keeps its flat data in ``_data``; here it is computed on demand
    @property
    def _data(self):
        if self._lazy is None:
            self._lazy = self._compute()
        return self._lazy

    @_data.setter
    def _data(self, v):
        self._lazy = v

    def is_materialised(self):
        return self._lazy is not None
