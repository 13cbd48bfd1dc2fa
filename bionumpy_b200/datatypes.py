"""Record containers for the chunk objects the readers yield: the field names of
bionumpy/datatypes/__init__.py:39-47 (SequenceEntry: name, sequence; SequenceEntryWithQuality:
+ quality), materialised lazily from the file buffer (bnpdataclass/lazybnpdataclass.py:117-125)."""
import numpy as np
import torch


def _from_strings(field, value):
    """Lists of Python strings, as the reference's dataclasses take them: names and sequences become text
    (as_encoded_array), quality strings byte - 33 (QualityEncoding, encodings/__init__.py:26)."""
    if not isinstance(value, list) or not all(isinstance(v, str) for v in value):
        return value
    if field == "quality":
        from .ragged import RaggedArray
        from . import config
        flat = np.frombuffer("".join(value).encode("ascii"), dtype=np.uint8) - np.uint8(33)
        data = torch.from_numpy(flat.copy()).to(config.default_device())
        return RaggedArray(data, [len(v) for v in value])
    from .encoded_array import as_encoded_array
    return as_encoded_array(value)


class _Entries:
    _fields = ()

    def __init__(self, *values, buffer=None):
        self._buffer = buffer
        self._values = {f: _from_strings(f, v) for f, v in zip(self._fields, values)}

    @classmethod
    def lazy(cls, buffer):
        return cls(buffer=buffer)

    def __getattr__(self, name):
        if name.startswith("_") or name not in self._fields:
            raise AttributeError(name)
        if name not in self._values:
            self._values[name] = self._buffer.get_field_by_number(self._fields.index(name))
        return self._values[name]

    def __getitem__(self, idx):
        """The selected entries (a bool mask, an index tensor/array/list or a slice): each field a view of the same
        bytes with the selected rows, no copy (``reads[np.sum(match_string(reads.sequence, "ACT"), axis=1) > 0]``)."""
        if isinstance(idx, (int, np.integer)):
            raise TypeError("select entries with a mask, an index array or a slice")
        if isinstance(idx, (list, np.ndarray)):
            idx = torch.as_tensor(np.asarray(idx))
        return self.__class__(*[getattr(self, f)[idx] for f in self._fields])

    def __len__(self):
        if self._buffer is not None:
            return self._buffer.count_entries()
        if not self._values:
            return 0
        return len(next(iter(self._values.values())))

    def __repr__(self):
        return f"{self.__class__.__name__} with {len(self)} entries"


def replace(entries, **fields):
    """dataclasses.replace for record chunks (bnpdataclass.py): the same record class, the named fields replaced and the
    others carried over."""
    unknown = set(fields) - set(entries._fields)
    if unknown:
        raise TypeError(f"{type(entries).__name__} has no field(s) {sorted(unknown)}")
    return type(entries)(*[fields[f] if f in fields else getattr(entries, f) for f in entries._fields])


def concatenate(a, b, extra=()):
    """The entries of ``a`` followed by those of ``b`` (np.concatenate of two records of one type), and the host values
    of ``extra`` (one-word device tensors, e.g. a kernel's output count), all read in one synchronisation.  Text
    fields are copied row by row (the flat mode of bnpk_interval_gather), so only the bytes of the rows, not the whole
    chunks they may be views of, are copied.  Returns (record, [extra values])."""
    if type(a) is not type(b):
        raise TypeError(f"cannot concatenate {type(a).__name__} and {type(b).__name__}")
    from . import ops
    from .encoded_array import EncodedArray, EncodedRaggedArray
    from .rows import RowView
    fields, texts, words = {}, {}, []
    for f in a._fields:
        x, y = getattr(a, f), getattr(b, f)
        if isinstance(x, EncodedRaggedArray) and isinstance(y, EncodedRaggedArray):
            if x.encoding != y.encoding:
                raise TypeError(f"the {f} fields have different encodings")
            texts[f] = [(RowView(v), ops.row_offsets(v._lens.contiguous())) for v in (x, y)]
            words += [offsets[-1:] for _, offsets in texts[f]]
        elif isinstance(x, EncodedArray) and isinstance(y, EncodedArray):
            fields[f] = EncodedArray(torch.cat([x.raw(), y.raw()]), x.encoding)
        elif isinstance(x, torch.Tensor) and isinstance(y, torch.Tensor):
            fields[f] = torch.cat([x, y])
        else:
            raise TypeError(f"cannot concatenate the {f} fields ({type(x).__name__}, {type(y).__name__})")
    values = torch.cat([w.to(torch.int64).reshape(1) for w in words + list(extra)]).cpu().tolist() if words or extra \
        else []
    for i, (f, parts) in enumerate(texts.items()):
        flat = [ops.interval_copy(rows.base, rows.starts, rows.starts + rows.lens.to(torch.int64), offsets, total)
                for (rows, offsets), total in zip(parts, values[2 * i:2 * i + 2])]
        x = getattr(a, f)
        fields[f] = EncodedRaggedArray(EncodedArray(torch.cat(flat), x.encoding),
                                       torch.cat([rows.lens for rows, _ in parts]))
    return type(a)(*[fields[f] for f in a._fields]), values[len(words):]


class SequenceEntry(_Entries):
    _fields = ("name", "sequence")


class SequenceEntryWithQuality(_Entries):
    _fields = ("name", "sequence", "quality")


class BamEntry(_Entries):
    """datatypes/__init__.py:173-183: an alignment.  chromosome and name are text, flag, position (0-based) and mapq
    int64 CUDA tensors, cigar_op CigarOpEncoding codes and cigar_length int64 per row, sequence BamEncoding codes and
    quality the stored phred values (uint8, 0xFF where the read has none)."""
    _fields = ("chromosome", "name", "flag", "position", "mapq", "cigar_op", "cigar_length", "sequence", "quality")


def _interval_field(field, value):
    """Interval, Bed6 and BedGraph fields: text columns (chromosome, name) as text, integer columns (start, stop, score)
    as int64 CUDA tensors, a bedGraph value as a CUDA tensor of its own dtype and strand as StrandEncoding codes."""
    if field in ("chromosome", "name"):
        return _from_strings(field, value)
    from . import config
    if field == "strand":
        from .encoded_array import EncodedArray
        from .encodings import StrandEncoding
        if isinstance(value, EncodedArray):
            return value
        if isinstance(value, str):
            value = list(value)
        codes = np.array(["+-.".index(v) for v in value], dtype=np.uint8)
        return EncodedArray(torch.from_numpy(codes).to(config.default_device()), StrandEncoding)
    if isinstance(value, torch.Tensor):
        return value
    if field == "value":
        return torch.as_tensor(np.asarray(value)).to(config.default_device())     # kept in its dtype
    if field == "score" and isinstance(value, list):
        value = [0 if v == "." else int(v) for v in value]        # Optional[int]: "." is 0 (io/strops.py:69-83)
    return torch.as_tensor(np.asarray(value, dtype=np.int64)).to(config.default_device())


class _IntervalEntries(_Entries):
    """Records whose fields can be assigned (``peaks.start = mid - 50``), as the reference's dataclasses allow."""

    def __init__(self, *values, buffer=None):
        super().__init__(buffer=buffer)
        for f, v in zip(self._fields, values):
            self._values[f] = _interval_field(f, v)

    def __setattr__(self, name, value):
        if name in self._fields:
            self._values[name] = _interval_field(name, value)
        else:
            super().__setattr__(name, value)

    @classmethod
    def from_entry_tuples(cls, tuples):
        """bnpdataclass.from_entry_tuples: one tuple per entry."""
        columns = list(zip(*tuples)) if len(tuples) else [[] for _ in cls._fields]
        return cls(*[list(c) for c in columns])


class Interval(_IntervalEntries):
    """datatypes/__init__.py:51-54: chromosome, start, stop (0-based, end-exclusive)."""
    _fields = ("chromosome", "start", "stop")


class StrandedInterval(_IntervalEntries):
    """datatypes/__init__.py:57-59: Interval + strand."""
    _fields = ("chromosome", "start", "stop", "strand")


class Bed6(_IntervalEntries):
    """datatypes/__init__.py:67-70: Interval + name, score (Optional[int]) and strand."""
    _fields = ("chromosome", "start", "stop", "name", "score", "strand")


class BedGraph(_IntervalEntries):
    """datatypes/__init__.py:27-31: chromosome, start, stop and value.  The value is an integer (or bool) tensor here:
    the tracks it comes from hold integers, and a float value cannot be written."""
    _fields = ("chromosome", "start", "stop", "value")
