"""NumPy restatement of the reference's position weight matrix code, for the motif tests (the package never imports it).

Each function cites the reference lines (bionumpy/ unless noted) it follows."""
import numpy as np

from oracle import bnp_oracle as o


def from_dict(dictionary, background=None):
    """PWM.from_dict, sequence/position_weight_matrix.py:102-130 -> (matrix [A, m], alphabet)."""
    if background is None:
        background = {key: 1 / len(dictionary) for key in dictionary}
    with np.errstate(divide="ignore"):
        matrix = np.log(np.array(list(dictionary.values()))) - \
            np.log([background[key] for key in dictionary])[:, np.newaxis]
    return matrix, "".join(dictionary.keys())


def from_counts(counts):
    """PWM.from_counts / _pwm_from_counts, sequence/position_weight_matrix.py:26-28,132-135."""
    c = np.array(list(counts.values())) + 1
    return np.log(c / c.sum(axis=0, keepdims=True)), "".join(counts.keys())


def read_jaspar(path):
    """read_jaspar_matrix, io/jaspar.py:5-16: the counts go to from_dict unchanged."""
    with open(path) as f:
        f.readline()
        d = {}
        for line in f:
            letter, rest = line.split(maxsplit=1)
            d[letter.strip()] = [float(n) for n in rest.strip()[1:-1].split()]
    return from_dict(d)


def read_csv(path):
    """read_csv_motif, io/jaspar.py:25-45."""
    with open(path) as f:
        alphabet = f.readline().strip().split(",")
        d = {a: [] for a in alphabet}
        for line in f:
            parts = line.strip().split(",")
            for i, a in enumerate(alphabet):
                d[a].append(float(parts[i]))
    return from_dict(d)


def pwm_str(matrix, alphabet):
    """PWM.__str__, sequence/position_weight_matrix.py:137-140 (the second definition, which wins)."""
    return "PWM with alphabet " + alphabet + "\n" + \
        "\n".join(" ".join(str(round(c, 2)) for c in row) for row in matrix.T)


def calculate_scores(codes, matrix):
    """PWM.calculate_scores, sequence/position_weight_matrix.py:83-100: zeros, then column by column in order; the last
    m - 1 positions keep the sums of the columns that fit."""
    codes = np.asarray(codes, dtype=np.int64)
    scores = np.zeros(codes.size, dtype=float)
    for offset, row in enumerate(matrix.T.copy()):
        scores[:scores.size - offset] += row[codes[offset:]]
    return scores


def motif_scores(codes_flat, lens, matrix):
    """get_motif_scores, sequence/position_weight_matrix.py:166-196: calculate_scores on the flattened rows, then the
    ragged [..., :-m+1].  m = 1 keeps every score (the one documented deviation).  Returns (flat scores, lens)."""
    flat = calculate_scores(codes_flat, matrix)
    return o.ragged_drop_tail(flat, np.asarray(lens, dtype=np.int64), matrix.shape[1] - 1)


def row_max(flat, lens):
    """scores.max(axis=-1) per row as np.max (NaN propagates); -inf for an empty row."""
    out = np.full(len(lens), -np.inf)
    pos = 0
    for r, L in enumerate(np.asarray(lens, dtype=np.int64)):
        if L:
            out[r] = np.max(flat[pos:pos + L])
        pos += L
    return out


def encode(byte_rows, alphabet):
    """Text rows -> codes with AlphabetEncoding(alphabet) (encodings/alphabet_encoding.py:19-46); the first bad flat
    offset or None."""
    lut = o.alphabet_lut(alphabet)
    flat = np.concatenate([np.frombuffer(r, dtype=np.uint8) for r in byte_rows]) if byte_rows else np.zeros(0, np.uint8)
    codes = lut[flat]
    bad = np.flatnonzero(codes == 255)
    return codes.astype(np.int64), (int(bad[0]) if bad.size else None)
