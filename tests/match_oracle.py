"""String and pattern matches restated with Python's ``re``: position p of a row matches iff
``re.match(pattern, row[p:], re.DOTALL)`` does.  Test infrastructure only; the package never imports it."""
import re

import numpy as np


class OracleEncodingError(Exception):
    def __init__(self, offset):
        super().__init__(f"invalid character at flat offset {offset}")
        self.offset = offset


def span(pattern, literal=False):
    """The longest expansion of a pattern: every class counts one column, a gap .{a,b} counts b."""
    if literal:
        return len(pattern)
    p = re.sub(r"\.\{(\d*),(\d+)\}", lambda g: "x" * int(g.group(2)), pattern)
    return len(re.sub(r"\[[^\]]*\]", "x", p))


def compile_pattern(pattern, literal=False, alphabet=None):
    """Bytes regex; ``literal`` escapes every character; ``alphabet`` (encoded input) upper-cases the letters."""
    if alphabet is not None:
        pattern = pattern.upper()
    return re.compile((re.escape(pattern) if literal else pattern).encode("latin-1"), re.DOTALL)


def prepare(rows, alphabet=None):
    """Rows (bytes) as the kernels read them: raw bytes as they are, encoded text upper-cased and validated
    (OracleEncodingError with the flat offset of the first byte outside the alphabet)."""
    if alphabet is None:
        return list(rows)
    ok = set(alphabet.upper().encode())
    out, flat = [], 0
    for r in rows:
        u = r.upper()
        for i, b in enumerate(u):
            if b not in ok:
                raise OracleEncodingError(flat + i)
        out.append(u)
        flat += len(r)
    return out


def matches(rows, pattern, mode="valid", literal=False, alphabet=None):
    """One list of bools per row: max(L - span + 1, 0) values ("valid") or L ("same")."""
    rx = compile_pattern(pattern, literal, alphabet)
    m = span(pattern, literal)
    out = []
    for r in prepare(rows, alphabet):
        n = len(r) if mode == "same" else max(len(r) - m + 1, 0)
        out.append([rx.match(r, p) is not None for p in range(n)])
    return out


def counts(rows, pattern, mode="valid", literal=False, alphabet=None):
    return np.array([sum(r) for r in matches(rows, pattern, mode, literal, alphabet)], dtype=np.int64)


def decode(codes, lens, alphabet):
    """Code rows back to letters (bytes), for encoded-array inputs."""
    letters = np.frombuffer(alphabet.encode(), dtype=np.uint8)
    flat = letters[np.asarray(codes, dtype=np.int64)]
    out, o = [], 0
    for n in lens:
        out.append(flat[o:o + n].tobytes())
        o += n
    return out
