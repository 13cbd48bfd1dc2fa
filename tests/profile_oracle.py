"""A plain-NumPy restatement of track profiles: locations of intervals, windows around them, clipping and extension
along the strand, dense tracks read back to front on '-' rows, the blocked column sum in the order include/bnpk.h
fixes, and narrowPeak rows read by float() and int()."""
import gzip

import numpy as np

BLOCK_ROWS = 256            # BNPK_COLUMN_BLOCK_ROWS
MINUS = "-"


# --------------------------------------------------------------------------------------------------------------------
# locations, windows, clip and extension (local coordinates; strand None for unstranded rows)
# --------------------------------------------------------------------------------------------------------------------
def location(start, stop, strand, where):
    """One row's 'start', 'stop' or 'center': on '-' the start is stop - 1 and the stop is start; on '+', '.' and
    unstranded rows the start is start and the stop is stop - 1; the center is (start + stop) // 2."""
    if where == "center":
        return (start + stop) // 2
    first, last = (start, stop - 1) if where == "start" else (stop - 1, start)
    return last if strand == MINUS else first


def clip(start, stop, size):
    return max(start, 0), min(stop, size)


def window(position, size, flank=None, window_size=None):
    """[p - flank, p + flank + 1), or [p - ws // 2, p + ws // 2 + ws % 2), clipped to [0, size)."""
    if flank is not None:
        left, right = flank, flank + 1
    else:
        left, right = window_size // 2, window_size // 2 + window_size % 2
    return clip(position - left, position + right, size)


def extended(start, stop, strand, length, size):
    """'+', '.' and unstranded rows keep their start, '-' rows their stop; then clipped."""
    if strand == MINUS:
        return clip(stop - length, stop, size)
    return clip(start, start + length, size)


# --------------------------------------------------------------------------------------------------------------------
# dense tracks, rows and column sums
# --------------------------------------------------------------------------------------------------------------------
def dense(run_starts, values):
    """The value at every position of runs [run_starts[i], run_starts[i + 1])."""
    run_starts = np.asarray(run_starts, dtype=np.int64)
    return np.repeat(np.asarray(values), np.diff(run_starts))


def rows(track, q_start, width, reverse=None):
    """The rows track[q : q + width], each reversed where reverse is true: an (N, width) matrix."""
    out = np.stack([track[q:q + width] for q in q_start]) if len(q_start) else np.zeros((0, width), track.dtype)
    if reverse is not None:
        flip = np.asarray(reverse, dtype=bool)
        out[flip] = out[flip, ::-1]
    return out


def column_sum(matrix):
    """The column sums of an (N, width) matrix in the fixed order: blocks of BLOCK_ROWS consecutive rows, each block's
    rows added in row order starting from +0.0, then the block partials added in block order starting from +0.0.
    Integer matrices are summed in int64, which wraps; float matrices in float64 (one rounding per add)."""
    kind = np.float64 if matrix.dtype.kind == "f" else np.int64
    m = matrix.astype(kind)
    width = m.shape[1]
    out = np.zeros(width, dtype=kind)
    with np.errstate(over="ignore", invalid="ignore"):
        for b in range(0, m.shape[0], BLOCK_ROWS):
            partial = np.zeros(width, dtype=kind)
            for row in m[b:b + BLOCK_ROWS]:
                partial = partial + row
            out = out + partial
    return out


def column_mean(matrix):
    """column_sum / N in float64 (an integer sum converted to float64 first)."""
    with np.errstate(invalid="ignore"):
        return column_sum(matrix).astype(np.float64) / matrix.shape[0]


# --------------------------------------------------------------------------------------------------------------------
# narrowPeak
# --------------------------------------------------------------------------------------------------------------------
def read_narrowpeak(path):
    """(chromosome, start, stop, name, score, strand, signal_value, p_value, q_value, summit) rows; score '.' is 0."""
    opener = gzip.open if str(path).endswith(".gz") else open
    out = []
    with opener(path, "rt") as f:
        for line in f:
            line = line.rstrip("\n")
            if not line or line.startswith("#"):
                continue
            c, s, e, name, score, strand, sv, pv, qv, summit = line.split("\t")[:10]
            out.append((c, int(s), int(e), name, 0 if score == "." else int(score), strand, float(sv), float(pv),
                        float(qv), int(summit)))
    return out
