"""A plain-Python restatement of bedGraph reading and float tracks: the decimal grammar checked by a regular expression
and read by float(), gaps filled with +0.0, the overlap rule, and exact per-interval sums (Fraction)."""
import math
import re
from fractions import Fraction

import numpy as np

GRAMMAR = re.compile(r"[+-]?(?:[0-9]+(?:\.[0-9]*)?|\.[0-9]+)(?:[eE][+-]?[0-9]+)?")
MAX_DIGITS = 19


def significant_digits(text):
    """The digits of the significand from its first to its last non-zero digit."""
    mantissa = re.split(r"[eE]", text.lstrip("+-"))[0].replace(".", "")
    stripped = mantissa.strip("0")
    return len(stripped)


def parse(text):
    """float(text) for text inside the grammar of at most 19 significant digits, else ValueError."""
    if not GRAMMAR.fullmatch(text) or significant_digits(text) > MAX_DIGITS:
        raise ValueError(f"not a bedGraph value: {text!r}")
    return float(text)


def is_header(line):
    return line.startswith("#") or line.startswith("track") or line.startswith("browser")


def read_bedgraph(path):
    """(chromosome, start, stop, value) rows after the leading header lines."""
    rows, body = [], False
    for line in open(path):
        line = line.rstrip("\n").rstrip("\r")
        if not body and is_header(line):
            continue
        body = True
        c, s, e, v = line.split("\t")[:4]
        rows.append((c, int(s), int(e), parse(v)))
    return rows


def read_sizes(path):
    return {line.split()[0]: int(line.split()[1]) for line in open(path) if line.strip()}


def read_bed(path):
    return [(c, int(s), int(e)) for c, s, e, *_ in (line.split("\t") for line in open(path) if line.strip())]


def dense_track(rows, sizes):
    """name -> float64 array: every row's value over [start, stop), +0.0 elsewhere.  Rows on unknown names raise
    KeyError, rows past their contig or with stop < start ValueError, overlapping rows ValueError."""
    out = {name: np.zeros(size, dtype=np.float64) for name, size in sizes.items()}
    covered = {name: np.zeros(size, dtype=bool) for name, size in sizes.items()}
    for c, s, e, v in rows:
        if c not in sizes:
            raise KeyError(c)
        if s < 0 or e < s or e > sizes[c]:
            raise ValueError(f"row {c}:{s}-{e} is not inside its contig")
        if covered[c][s:e].any():
            raise ValueError(f"row {c}:{s}-{e} overlaps an earlier row")
        covered[c][s:e] = True
        out[c][s:e] = v
    return out


def interval_max(dense, intervals):
    return [float(np.max(dense[c][s:e])) if e > s else -math.inf for c, s, e in intervals]


def exact_sum(values):
    """The sum of finite float values, exactly, as a Fraction (math.fsum rounds it once)."""
    return sum((Fraction(float(v)) for v in values), Fraction(0))


def interval_mean(dense, intervals):
    return [float(exact_sum(dense[c][s:e]) / (e - s)) if e > s else math.nan for c, s, e in intervals]
