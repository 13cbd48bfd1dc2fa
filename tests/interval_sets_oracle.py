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
