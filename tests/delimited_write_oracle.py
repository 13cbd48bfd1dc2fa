"""NumPy restatement of the reference's delimited writing and of a track's rows, for the write and track-interval tests
(the package never imports it).  Tracks enter as dense arrays per contig: the runs under test are never read.

Each function cites the reference lines (bionumpy/ unless noted) it follows."""
import numpy as np

STRANDS = b"+-."


def ints_to_strings(values):
    """io/strops.py ints_to_strings: decimal, '-' for a negative value, no leading zero."""
    return [str(int(v)).encode() for v in np.asarray(values, dtype=np.int64)]


def dump_lines(columns):
    """io/dump_csv.py dump_csv + io/strops.py:186-215 join_columns: every column formatted, the columns of a line
    joined by '\\t' and every line ended by '\\n'.  A column is ("text", list of bytes), ("int", ints) or ("strand",
    StrandEncoding codes)."""
    cols = []
    for kind, data in columns:
        if kind == "text":
            cols.append([x.encode() if isinstance(x, str) else bytes(x) for x in data])
        elif kind == "int":
            cols.append(ints_to_strings(data))
        else:
            cols.append([STRANDS[min(int(c), 2):min(int(c), 2) + 1] for c in data])
    n = {len(c) for c in cols}
    assert len(n) == 1, n
    return b"".join(b"\t".join(fields) + b"\n" for fields in zip(*cols))


def bed_columns(chroms, starts, stops):
    return [("text", [c.encode() if isinstance(c, str) else c for c in chroms]), ("int", starts), ("int", stops)]


def _runs(dense):
    """(starts, ends, values) of the maximal runs of equal value of one dense array."""
    dense = np.asarray(dense)
    if dense.size == 0:
        return (np.zeros(0, np.int64),) * 2 + (dense[:0],)
    change = np.flatnonzero(dense[1:] != dense[:-1]) + 1
    starts = np.concatenate([[0], change]).astype(np.int64)
    ends = np.concatenate([change, [dense.size]]).astype(np.int64)
    return starts, ends, dense[starts]


def nonzero_intervals(dense_by_contig):
    """GenomicIntervals.from_track as its docstring states it (genomic_data/genomic_intervals.py:529-543): the maximal
    stretches of non-zero value of every contig, in the order given.  Returns (names, starts, stops)."""
    names, starts, stops = [], [], []
    for name, dense in dense_by_contig.items():
        s, e, v = _runs(np.asarray(dense) != 0)
        keep = v.astype(bool)
        names += [name] * int(keep.sum())
        starts.append(s[keep])
        stops.append(e[keep])
    cat = (lambda xs: np.concatenate(xs) if xs else np.zeros(0, np.int64))
    return names, cat(starts), cat(stops)


def bedgraph_rows(dense_by_contig):
    """GenomicArrayGlobal.get_data / _get_intervals_from_data (genomic_data/genomic_track.py:84-91,199-218) of a
    canonical track: every run of every contig with its value.  Returns (names, starts, stops, values)."""
    names, starts, stops, values = [], [], [], []
    for name, dense in dense_by_contig.items():
        s, e, v = _runs(dense)
        names += [name] * len(s)
        starts.append(s)
        stops.append(e)
        values.append(np.asarray(v).astype(np.int64))
    cat = (lambda xs: np.concatenate(xs) if xs else np.zeros(0, np.int64))
    return names, cat(starts), cat(stops), cat(values)


def dense_of_rows(names, starts, stops, values, sizes, dtype=np.int64):
    """The dense arrays per contig that rows (names, local [start, stop), value) describe; positions no row covers are
    0.  Raises AssertionError if two rows overlap."""
    out = {n: np.zeros(s, dtype=dtype) for n, s in sizes.items()}
    seen = {n: np.zeros(s, dtype=bool) for n, s in sizes.items()}
    for n, a, b, v in zip(names, starts, stops, values):
        assert not seen[n][a:b].any(), (n, a, b)
        seen[n][a:b] = True
        out[n][a:b] = v
    return out
