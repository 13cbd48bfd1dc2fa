"""Similarity of two interval sets over a genome (mirror of bionumpy/arithmetics/similarity_measures.py): the
contingency table of their masks, the Forbes and the Jaccard index.

The masks are run-length tracks on the device (get_boolean_mask / GenomicIntervals.get_mask), their intersection is one
bnpk_runs_combine, and the three sums come back in one copy; the final formula is evaluated on Python integers, so
a * N does not overflow on genome-sized inputs.  The intervals need not be sorted."""
import torch

from ..genomic_data.genome import Genome
from .intervals import get_boolean_mask


def _table(a, b, ab, n):
    return [[ab, a - ab], [b - ab, n - a - b + ab]]


def get_contingency_table(intervals_a, intervals_b, sequence_length):
    """[[both, only a], [only b, neither]]: the positions of one contig of ``sequence_length`` covered by both interval
    sets, by one of them or by none."""
    mask_a = get_boolean_mask(intervals_a, sequence_length)
    mask_b = get_boolean_mask(intervals_b, sequence_length)
    sums = torch.stack([mask_a.sum(), mask_b.sum(), (mask_a & mask_b).sum()]).cpu().tolist()
    return _table(*sums, int(sequence_length))


def _genome_table(chromosome_sizes, intervals_a, intervals_b):
    """The contingency table over every contig of ``chromosome_sizes`` (a {name: size} dict, all contigs kept, or a
    Genome); an interval on a name outside it raises KeyError."""
    genome = chromosome_sizes if isinstance(chromosome_sizes, Genome) else \
        Genome(dict(chromosome_sizes), filter_function=None)
    mask_a = genome.get_intervals(intervals_a).get_mask()
    mask_b = genome.get_intervals(intervals_b).get_mask()
    sums = torch.stack([mask_a.sum(), mask_b.sum(), (mask_a & mask_b).sum()]).cpu().tolist()
    return _table(*sums, genome.size)


def forbes(chromosome_sizes, intervals_a, intervals_b) -> float:
    """The Forbes similarity index N * |a & b| / (|a| * |b|) of two interval sets.

    >>> a = Interval.from_entry_tuples([("chr1", 10, 20), ("chr2", 20, 30)])
    >>> b = Interval.from_entry_tuples([("chr2", 15, 25), ("chr1", 10, 40)])
    >>> forbes({"chr1": 100, "chr2": 200}, a, b)
    5.625"""
    ((a, b), (c, d)) = _genome_table(chromosome_sizes, intervals_a, intervals_b)
    n = a + b + c + d
    return float(a * n / ((a + b) * (a + c)))


def jaccard(chromosome_sizes, intervals_a, intervals_b) -> float:
    """The Jaccard similarity index |a & b| / |a | b| of two interval sets."""
    ((a, b), (c, d)) = _genome_table(chromosome_sizes, intervals_a, intervals_b)
    n = a + b + c + d
    return float(a / (n - d))
