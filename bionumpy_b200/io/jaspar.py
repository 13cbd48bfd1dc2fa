"""Motif files: JASPAR count matrices and CSV probability matrices (mirror of bionumpy/io/jaspar.py:5-45).

Both pass their values straight to PWM.from_dict, as the reference does: a JASPAR file's counts become
log(count) - log(1 / alphabet size), not normalised probabilities."""
from ..sequence.position_weight_matrix import PWM


def parse_jaspar_line(line):
    """'A  [ 14 4 3 ]' -> ('A', [14.0, 4.0, 3.0])."""
    letter, rest = line.split(maxsplit=1)
    counts = [float(n) for n in rest.strip()[1:-1].split()]
    return letter.strip(), counts


def read_jaspar_matrix(filename) -> PWM:
    """A JASPAR matrix: a '>' header line, then one 'letter [counts]' line per letter."""
    with open(filename) as f:
        f.readline()
        pwm = dict(parse_jaspar_line(line) for line in f if line.strip())
    return PWM.from_dict(pwm)


def read_csv_motif(filename) -> PWM:
    """A CSV motif: the alphabet on the first line, then one line of probabilities per motif position."""
    with open(filename) as f:
        alphabet = f.readline().strip().split(",")
        pwm = {letter: [] for letter in alphabet}
        for line in f:
            if not line.strip():
                continue
            parts = line.strip().split(",")
            for i, letter in enumerate(alphabet):
                pwm[letter].append(float(parts[i]))
    return PWM.from_dict(pwm)
