"""NumPy restatement of the reference's pileups, masks, merges and genome layout (bionumpy/arithmetics/intervals.py:137-304,
genomic_data/genome.py, genome_context.py).  Test infrastructure only: the package never imports it."""
import numpy as np


def dense_pileup(starts, stops, size):
    """tests/test_pileup.py raw_pileup: +1 over [start, stop) for every interval."""
    diff = np.zeros(size + 1, dtype=np.int64)
    np.add.at(diff, np.asarray(starts, dtype=np.int64), 1)
    np.add.at(diff, np.asarray(stops, dtype=np.int64), -1)
    return np.cumsum(diff)[:size]


def dense_mask(starts, stops, size):
    """tests/test_intervals.py::test_get_boolean_mask: true[start:end] |= True."""
    out = np.zeros(size, dtype=bool)
    for a, b in zip(starts, stops):
        out[a:b] = True
    return out


def runs_of(dense):
    """The canonical runs of a dense array: (starts, ends, values), no two neighbouring runs with the same value."""
    dense = np.asarray(dense)
    if dense.size == 0:
        return np.zeros(0, np.int64), np.zeros(0, np.int64), dense[:0]
    change = np.flatnonzero(dense[1:] != dense[:-1]) + 1
    starts = np.concatenate([[0], change]).astype(np.int64)
    ends = np.concatenate([change, [dense.size]]).astype(np.int64)
    return starts, ends, dense[starts]


def event_runs(starts, stops, size, any_mode=False):
    """The same runs from the events alone (sizes too large for a dense array): the coverage after every distinct
    position, neighbours with equal values merged."""
    starts, stops = np.asarray(starts, dtype=np.int64), np.asarray(stops, dtype=np.int64)
    pos = np.concatenate([starts, stops, [0]])
    delta = np.concatenate([np.ones(starts.size, np.int64), -np.ones(stops.size, np.int64), [0]])
    order = np.argsort(pos, kind="stable")
    pos, delta = pos[order], delta[order]
    cov = np.cumsum(delta)
    last = np.concatenate([pos[1:] != pos[:-1], [True]])
    p, v = pos[last], cov[last]
    keep = p < size
    p, v = p[keep], v[keep]
    if any_mode:
        v = v > 0
    change = np.concatenate([[True], v[1:] != v[:-1]])
    p, v = p[change], v[change]
    return p, np.concatenate([p[1:], [size]]).astype(np.int64), v


def reduce_runs(run_starts, run_ends, values, a, b, how):
    """max / min / sum / any of the track over [a, b) for every query, from the runs; empty queries follow
    RaggedArray (segment_max: INT64_MIN, segment_min: INT64_MAX, sum 0, any False)."""
    out = []
    for s, e in zip(a, b):
        lo = np.searchsorted(run_starts, s, side="right") - 1
        hi = np.searchsorted(run_starts, e, side="left")
        if e <= s:
            out.append({"max": np.iinfo(np.int64).min, "min": np.iinfo(np.int64).max, "sum": 0, "any": False}[how])
            continue
        v = np.asarray(values[lo:hi], dtype=np.int64)
        overlap = np.minimum(run_ends[lo:hi], e) - np.maximum(run_starts[lo:hi], s)
        out.append({"max": v.max(), "min": v.min(), "sum": int((v * overlap).sum()), "any": bool((v != 0).any())}[how])
    return np.array(out)


def dense_of(starts, ends, values, dtype=None):
    """The dense array of a track given by its runs (the inverse of runs_of), in ``dtype`` (default the values')."""
    values = np.asarray(values)
    counts = np.asarray(ends, dtype=np.int64) - np.asarray(starts, dtype=np.int64)
    return np.repeat(values.astype(dtype or values.dtype), counts)


def extremes(dtype):
    """Values a track of ``dtype`` must survive: both ends of its range, their neighbours, -1, 0 and 1."""
    dtype = np.dtype(dtype)
    if dtype == np.bool_:
        return np.array([False, True])
    info = np.iinfo(dtype)
    vals = {info.min, info.min + 1, info.max - 1, info.max, 0, 1} | ({-1} if info.min < 0 else set())
    return np.array(sorted(vals), dtype=dtype)


def random_dense(rng, size, dtype, max_run=4):
    """A dense track of ``size`` positions in runs of 1..max_run equal values: half of the runs take a value of
    extremes(dtype), the rest a random value of the whole range (neighbouring runs may be equal)."""
    dtype = np.dtype(dtype)
    lens = rng.integers(1, max_run + 1, size + 1)
    n_runs = int(np.searchsorted(np.cumsum(lens), size)) + 1
    lens = lens[:n_runs]
    if dtype == np.bool_:
        vals = rng.integers(0, 2, n_runs).astype(bool)
    else:
        info = np.iinfo(dtype)
        vals = rng.integers(info.min, info.max, n_runs, dtype=dtype, endpoint=True)
        pick = rng.integers(0, 2, n_runs).astype(bool)
        ext = extremes(dtype)
        vals[pick] = ext[rng.integers(0, ext.size, int(pick.sum()))]
    return np.repeat(vals, lens)[:size]


def empty_value(how, dtype):
    """What a reduction gives for a row with no values (RaggedArray's rule): max the dtype's lowest value and min its
    highest (False / True for bool), sum 0, mean NaN, any False."""
    dtype = np.dtype(dtype)
    if how in ("max", "min"):
        if dtype == np.bool_:
            return how == "min"
        info = np.iinfo(dtype)
        return info.min if how == "max" else info.max
    return {"sum": 0, "mean": np.nan, "any": False}[how]


def clip_queries(a, b, size):
    """[a, b) clipped to [0, size) as the run-length arrays clip them: a to [0, size], b to [a, size]."""
    a = np.clip(np.asarray(a, dtype=np.int64), 0, size)
    b = np.minimum(np.maximum(np.asarray(b, dtype=np.int64), a), size)
    return a, b


def reduce_dense(dense, a, b, how):
    """max / min / sum / mean / any of ``dense`` over [a, b) for every query, each query clipped to [0, size) first,
    from the dense values alone (never the runs).  Vectorised: prefix sums for sum / mean / any and
    np.maximum.reduceat / np.minimum.reduceat for max / min, so millions of queries and positions take well under a
    second.  max / min keep the track's dtype; sum is int64 and wraps modulo 2^64 as the kernels do (NumPy's int64
    array arithmetic wraps silently), so comparing int64 values compares the sums modulo 2^64; mean is float64 of that
    int64 sum over the length, which is the true mean, rounded once, only where the true sum is below 2^53 in
    magnitude (mean_is_exact); any is bool.  Empty rows give empty_value(how, dense.dtype)."""
    dense = np.asarray(dense)
    a, b = clip_queries(a, b, dense.size)
    empty = b <= a
    if how in ("max", "min"):
        # a uint8 view of bool keeps reduceat to plain integer code; one spare element keeps every index in range
        work = dense.view(np.uint8) if dense.dtype == np.bool_ else dense
        work = np.concatenate([work, work[:1] if work.size else np.zeros(1, work.dtype)])
        ufunc = np.maximum if how == "max" else np.minimum
        got = ufunc.reduceat(work, np.stack([a, b], 1).reshape(-1))[0::2] if a.size else work[:0]
        got = got.astype(dense.dtype)
        got[empty] = empty_value(how, dense.dtype)
        return got
    if how == "any":
        nonzero = np.concatenate([[0], np.cumsum(dense != 0, dtype=np.int64)])
        return nonzero[b] - nonzero[a] > 0
    prefix = np.concatenate([[0], np.cumsum(dense.astype(np.int64), dtype=np.int64)])
    total = prefix[b] - prefix[a]
    if how == "sum":
        return total
    with np.errstate(invalid="ignore", divide="ignore"):
        return total.astype(np.float64) / (b - a).astype(np.float64)


def mean_is_exact(dense, a, b):
    """Where the mean of reduce_dense is exact: the sum of |value| over the clipped row is below 2^52 (a float64
    running sum of the row, in any order, is then exact too)."""
    dense = np.asarray(dense)
    a, b = clip_queries(a, b, dense.size)
    mag = np.concatenate([[0.0], np.cumsum(np.abs(dense.astype(np.float64)))])
    return mag[b] - mag[a] < 2.0 ** 52


def reduce_loop(dense, a, b, how):
    """reduce_dense as a plain loop over the positions of every query, sums in exact Python integers reduced
    modulo 2^64 to int64 at the end."""
    dense = np.asarray(dense)
    out = []
    for s, e in zip(*clip_queries(a, b, dense.size)):
        vals = [int(v) for v in dense[s:e]]
        if not vals:
            out.append(empty_value(how, dense.dtype))
        elif how == "max":
            out.append(max(vals))
        elif how == "min":
            out.append(min(vals))
        elif how == "any":
            out.append(any(v != 0 for v in vals))
        else:
            total = sum(vals)
            wrapped = (total + 2 ** 63) % 2 ** 64 - 2 ** 63
            out.append(wrapped if how == "sum" else float(np.float64(wrapped) / np.float64(len(vals))))
    return out


def merge_intervals(starts, stops, distance=0):
    """arithmetics/intervals.py:270-304 line by line, on one chromosome: (kept row indices, merged stops)."""
    starts, stops = np.asarray(starts, dtype=np.int64), np.asarray(stops, dtype=np.int64)
    if starts.size == 0:
        return np.zeros(0, np.int64), np.zeros(0, np.int64)
    assert np.all(starts[:-1] <= starts[1:]), "merge_intervals requires intervals sorted on start position"
    s = np.maximum.accumulate(stops)
    if distance > 0:
        s = s + distance
    valid_start_mask = starts[1:] > s[:-1]
    start_mask = np.concatenate(([True], valid_start_mask))
    stop_mask = np.concatenate((valid_start_mask, [True]))
    new_stop = s[stop_mask]
    if distance > 0:
        new_stop = new_stop - distance
    return np.flatnonzero(start_mask), new_stop


def merge_by_chromosome(chroms, starts, stops, distance=0):
    """chromosome_map: merge every block of consecutive rows with one chromosome name."""
    chroms = list(chroms)
    rows, out_stops = [], []
    i = 0
    while i < len(chroms):
        j = i
        while j < len(chroms) and chroms[j] == chroms[i]:
            j += 1
        r, s = merge_intervals(starts[i:j], stops[i:j], distance)
        rows.extend((r + i).tolist())
        out_stops.extend(s.tolist())
        i = j
    return np.array(rows, dtype=np.int64), np.array(out_stops, dtype=np.int64)


def read_sizes(text):
    out = {}
    for line in text.splitlines():
        parts = line.split()
        if len(parts) >= 2:
            out[parts[0]] = int(parts[1])
    return out


def genome_layout(sizes, filter_function=lambda name: "_" not in name):
    """genome_context.py: the included contigs in file order and each one's global offset."""
    names = [n for n in sizes if filter_function(n)]
    offsets = np.concatenate([[0], np.cumsum([sizes[n] for n in names])]).astype(np.int64)
    return names, dict(zip(names, offsets[:-1].tolist())), int(offsets[-1])


def genome_intervals(sizes, chroms, starts, stops, filter_function=lambda name: "_" not in name):
    """Genome.get_intervals: rows on left-out contigs dropped, the rest with global coordinates; an unknown name
    raises KeyError and an interval outside its contig ValueError.  Returns (kept rows, global starts, global stops)."""
    names, offsets, _ = genome_layout(sizes, filter_function)
    keep, gs, ge = [], [], []
    for r, (c, a, b) in enumerate(zip(chroms, starts, stops)):
        if c not in sizes:
            raise KeyError(c)
        if c not in offsets:
            continue
        if a < 0 or b < a or b > sizes[c]:
            raise ValueError(r)
        keep.append(r)
        gs.append(offsets[c] + a)
        ge.append(offsets[c] + b)
    return np.array(keep, dtype=np.int64), np.array(gs, dtype=np.int64), np.array(ge, dtype=np.int64)


def contig_runs(run_starts, run_ends, values, offset, size):
    """The runs of one contig of a global track, clipped to it (local coordinates)."""
    lo = np.searchsorted(run_starts, offset, side="right") - 1
    hi = np.searchsorted(run_starts, offset + size, side="left")
    s = np.clip(run_starts[lo:hi] - offset, 0, size)
    e = np.clip(run_ends[lo:hi] - offset, 0, size)
    return s, e, values[lo:hi]


def parse_bed(text):
    """chromosome, start, stop of every line of BED text."""
    chroms, starts, stops = [], [], []
    for line in text.decode().splitlines():
        if not line or line.startswith("#"):
            continue
        f = line.split("\t")
        chroms.append(f[0])
        starts.append(int(f[1]))
        stops.append(int(f[2]))
    return chroms, np.array(starts, dtype=np.int64), np.array(stops, dtype=np.int64)
