"""The powers of five the device decimal parser needs (bnpk_parse_float): computed once per device on the host with
exact Python integers, as Eisel-Lemire's table is defined (Lemire, "Number parsing at a gigabyte per second", 2021)."""
import numpy as np

from .. import _native as nv

_tables = {}


def pow5_words():
    """uint64[2 * 651]: for q = -342 .. 308 the high and low words of 5^q truncated to 128 bits with bit 127 set.  For
    q < 0 the word is floor(2^b / 5^-q) + 1, truncated to 128 bits, with b = z + 127 for q >= -27 and 2z + 128 below
    (z the bit length of 5^-q), so that it is never below the true value's leading 128 bits."""
    words = []
    for q in range(nv.POW5_MIN, nv.POW5_MAX + 1):
        if q < 0:
            p = 5 ** -q
            z = p.bit_length()
            c = (1 << (z + 127 if q >= -27 else 2 * z + 128)) // p + 1
            c >>= max(c.bit_length() - 128, 0)
        else:
            c = 5 ** q
            n = c.bit_length()
            c = c << (128 - n) if n < 128 else c >> (n - 128)
        words += [c >> 64, c & ((1 << 64) - 1)]
    return np.array(words, dtype=np.uint64)


def pow5_table(device):
    """pow5_words() on ``device`` as int64 (the words' bits), built once per device."""
    if device not in _tables:
        from ..arithmetics.intervals import to_device
        _tables[device] = to_device(pow5_words().view(np.int64), device)
    return _tables[device]
