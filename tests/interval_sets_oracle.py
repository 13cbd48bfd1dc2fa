"""NumPy restatement of the reference's interval-set functions (bionumpy/arithmetics/intervals.py:235-342,
similarity_measures.py) and a dense oracle for the operators between run-length tracks.  Intervals are given as
(chromosome names, starts, stops); results are row indices into the concatenation the reference builds, so that a test
can compare every row and every field.  Test infrastructure only: the package never imports it."""
import numpy as np

import pileup_oracle as po


def _cat(a, b):
    return (list(a[0]) + list(b[0]), np.concatenate([a[1], b[1]]).astype(np.int64),
            np.concatenate([a[2], b[2]]).astype(np.int64))


def sweep(starts, stops):
    """The sorted sweep of intersect (intervals.py:317-325): (rows of the input, their new stops), in sweep order."""
    order = np.argsort(starts, kind="mergesort")
    s = np.asarray(starts)[order]
    e = np.sort(stops, kind="mergesort")
    mask = e[:-1] > s[1:]
    return order[1:][mask], e[:-1][mask]


def intersect(a, b):
    """intersect(a, b): rows of concatenate([a, b]) and their stops; the chromosome is ignored, as the reference does."""
    _, s, e = _cat(a, b)
    return sweep(s, e)


def global_intersect(b, a):
    """global_intersect(b, a) (intervals.py:328-335) on the rows of concatenate([a, b]), ordered by (name as bytes,
    start) and stops by (name, stop), with one change from the reference: no pair crosses a change of chromosome."""
    names, s, e = _cat(a, b)
    key = np.array([n.encode() for n in names], dtype=object)
    rank = np.unique(key, return_inverse=True)[1].reshape(-1) if len(names) else np.zeros(0, np.int64)
    order = np.lexsort((s, rank))
    stops = e[np.lexsort((e, rank))]
    r = rank[order]
    mask = (stops[:-1] > s[order][1:]) & (r[1:] == r[:-1])
    return order[1:][mask], stops[:-1][mask]


def count_overlap(a, b):
    """count_overlap (intervals.py:307-314) on one contig."""
    s = np.sort(np.concatenate([a[1], b[1]]), kind="mergesort")
    e = np.sort(np.concatenate([a[2], b[2]]), kind="mergesort")
    return int(np.sum(np.maximum(e[:-1] - s[1:], 0)))


def merged_by_chromosome(chroms, starts, stops):
    """{name: (merged starts, merged stops)}: the union of the intervals of every chromosome."""
    out = {}
    chroms = np.asarray(chroms, dtype=object)
    for name in set(chroms.tolist()):
        sel = chroms == name
        s, e = np.asarray(starts)[sel], np.asarray(stops)[sel]
        keep = e > s
        s, e = s[keep], e[keep]
        order = np.argsort(s, kind="mergesort")
        s, e = s[order], np.maximum.accumulate(e[order]) if s.size else e
        if s.size == 0:
            out[name] = (s, e)
            continue
        new = np.concatenate([[True], s[1:] > e[:-1]])
        last = np.concatenate([new[1:], [True]])
        out[name] = (s[new], e[last])
    return out


def unique_intersect(a, b):
    """unique_intersect (intervals.py:338-342) on whole genomes: the rows of a whose [start, stop) meets an interval of b
    on the same chromosome."""
    union = merged_by_chromosome(*b)
    keep = []
    for r, (c, s, e) in enumerate(zip(a[0], a[1], a[2])):
        if c not in union or e <= s:
            continue
        ms, me = union[c]
        i = np.searchsorted(me, s, side="right")
        if i < ms.size and ms[i] < e:
            keep.append(r)
    return np.array(keep, dtype=np.int64)


def sort_intervals(chroms, starts, stops, key=lambda x: x, sort_order=None):
    """sort_intervals (intervals.py:235-256): row order by (key(name), start, stop, row)."""
    if sort_order is not None:
        key = {name: i for i, name in enumerate(sort_order)}.__getitem__
    s = sorted((key(c), int(a), int(b), i) for i, (c, a, b) in enumerate(zip(chroms, starts, stops)))
    return np.array([t[-1] for t in s], dtype=np.int64)


def covered(chroms, starts, stops):
    return sum(int((e - s).sum()) for s, e in merged_by_chromosome(chroms, starts, stops).values())


def contingency_table(a, b, n):
    """get_contingency_table summed over contigs of total size n: [[a & b, a & ~b], [~a & b, ~a & ~b]]."""
    ca, cb = covered(*a), covered(*b)
    cab = ca + cb - covered(*_cat(a, b))
    return [[cab, ca - cab], [cb - cab, n - ca - cb + cab]]


def forbes(sizes, a, b):
    ((x, y), (z, w)) = contingency_table(a, b, sum(sizes.values()))
    n = x + y + z + w
    return float(x * n / ((x + y) * (x + z)))


def jaccard(sizes, a, b):
    ((x, y), (z, w)) = contingency_table(a, b, sum(sizes.values()))
    return float(x / (x + y + z))


# --------------------------------------------------------------------------------------------------------------------
# track operators
# --------------------------------------------------------------------------------------------------------------------
def widen(x):
    """What the tracks compute on: bool stays bool, every integer type becomes int64; scalars are kept."""
    if isinstance(x, np.ndarray):
        return x if x.dtype == np.bool_ else x.astype(np.int64)
    return x


def dense_op(ufunc, *operands):
    """The ufunc on the dense arrays (narrow integers widened to int64), and its canonical runs."""
    with np.errstate(over="ignore"):
        out = ufunc(*[widen(x) for x in operands])
    return out, po.runs_of(out)


ITEMS = {"a": 1, "b": 1, "ab": 2}


def event_tracks(events, at, m, after=0, seed=0):
    """Two tracks A and B laid out by events, the first merged run start of ``events[at]`` at merged index ``m``.

    Merged order is the combine kernel's: run starts by position, an A start before a B start at one position.  Each
    event is (side, a, b) at a position of its own: side "a", "b" or "ab" starts a run of A, of B or of both there, and
    a and b are the values from there on (the value of a side that starts no run is ignored; a value equal to the one
    before gives equal neighbouring runs, as astype does).  Position 0 holds both first runs (merged indices 0 and 1),
    filler events of random sides and changing values take the merged indices up to the events, and filler events of
    exactly ``after`` merged run starts follow them.  Gaps between positions are 1 to 3.  The placement is asserted
    against a plain sort of the starts.  Returns ((a_starts, a_ends, a_values), (b_starts, b_ends, b_values), size),
    int64, and the event's position."""
    rng = np.random.default_rng(seed)
    before = m - 2 - sum(ITEMS[e[0]] for e in events[:at])
    assert before >= 0, (m, events[:at])
    code = {"a": 1, "b": 2, "ab": 3}                 # bit 0: A starts a run, bit 1: B does

    def filler(n_items):
        """Random sides whose run starts number exactly n_items (a last tie that would overshoot becomes an A)."""
        sides = rng.integers(1, 4, n_items + 1)
        items = np.cumsum(np.where(sides == 3, 2, 1))
        k = int(np.searchsorted(items, n_items))
        sides = sides[:k + 1] if n_items else sides[:0]
        if n_items and items[k] > n_items:
            sides[k] = 1
        return sides

    head, tail = filler(before), filler(after)
    sides = np.concatenate([[3], head, [code[e[0]] for e in events], tail]).astype(np.int64)
    n, first = sides.size, 1 + head.size
    pos = np.concatenate([[0], np.cumsum(rng.integers(1, 4, n - 1))]).astype(np.int64)
    size = int(pos[-1]) + int(rng.integers(1, 4))
    out = []
    for k in range(2):
        # filler values change by 1..3 modulo 7 at every start, so filler runs are canonical; the events' values
        # are set as given and the fillers after them go on from the last one
        step = np.where(sides >> k & 1 == 1, rng.integers(1, 4, n), 0)
        vals = np.zeros(n, dtype=np.int64)
        vals[:first] = (int(rng.integers(0, 7)) + np.cumsum(step[:first])) % 7
        mine = sides[:first] >> k & 1 == 1
        last = int(vals[:first][mine][-1])
        for i, e in enumerate(events):
            vals[first + i] = e[1 + k] if sides[first + i] >> k & 1 else last
            last = int(vals[first + i])
        vals[first + len(events):] = (last + np.cumsum(step[first + len(events):])) % 7
        sel = sides >> k & 1 == 1
        starts = pos[sel]
        out.append((starts, np.append(starts[1:], size).astype(np.int64), vals[sel]))
    mp = np.concatenate([out[0][0], out[1][0]])
    side = np.concatenate([np.zeros(out[0][0].size, np.int64), np.ones(out[1][0].size, np.int64)])
    order = np.lexsort((side, mp))
    p = int(pos[first + at])
    assert (mp[order[m]], side[order[m]]) == (p, 0 if "a" in events[at][0] else 1), (m, p)
    assert mp.size == m + sum(ITEMS[e[0]] for e in events[at:]) + after
    return out[0], out[1], size, p


def sweep_loop(start, stop, same_prev=None):
    """bnpk_interval_intersect as a loop over the rows as given: row i is emitted iff i > 0, same_prev[i] (when given)
    and stop[i - 1] > start[i], with stop[i - 1] as its stop.  Returns (rows, stops, overlap): overlap is the sum of
    stop[i - 1] - start[i] over the emitted rows in exact integers, wrapped to int64 as NumPy's int64 sum wraps."""
    rows, stops, total = [], [], 0
    for i in range(1, len(start)):
        if (same_prev is None or same_prev[i]) and int(stop[i - 1]) > int(start[i]):
            rows.append(i)
            stops.append(int(stop[i - 1]))
            total += int(stop[i - 1]) - int(start[i])
    return np.array(rows, dtype=np.int64), np.array(stops, dtype=np.int64), (total + 2 ** 63) % 2 ** 64 - 2 ** 63


def mask_intersect(a, b):
    """The true intersection of two interval sets from dense masks, never the sweep: {name: (starts, stops)}, the
    runs where both sets cover, on every chromosome of either set (each as long as its largest stop)."""
    out = {}
    for name in sorted(set(a[0]) | set(b[0])):
        sel = [(np.asarray(x[0], dtype=object) == name) for x in (a, b)]
        size = max([int(np.max(x[2][s])) for x, s in zip((a, b), sel) if s.any()] + [0])
        both = po.dense_mask(a[1][sel[0]], a[2][sel[0]], size) & po.dense_mask(b[1][sel[1]], b[2][sel[1]], size)
        s, e, v = po.runs_of(both)
        out[name] = (s[v], e[v])
    return out
