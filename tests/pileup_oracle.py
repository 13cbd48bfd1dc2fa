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
