"""read_motif: a motif file by its suffix (mirror of bionumpy/io/motifs.py:1-20)."""
from dataclasses import dataclass
from pathlib import PurePath

import numpy as np

from .jaspar import read_jaspar_matrix, read_csv_motif

parsers = {".jaspar": read_jaspar_matrix, ".csv": read_csv_motif}


@dataclass
class Motif:
    alphabet: str
    matrix: np.ndarray


def read_motif(filename):
    """A PWM from a .jaspar or .csv file."""
    suffix = PurePath(filename).suffixes[-1]
    return parsers[suffix](filename)
