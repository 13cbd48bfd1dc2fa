"""Interval arithmetics on the device (bionumpy/arithmetics): pileups, masks and merges of the intervals of one
contig."""
from .intervals import (GenomicRunLengthArray, RunsRaggedArray, get_pileup, get_boolean_mask, merge_intervals)

__all__ = ["GenomicRunLengthArray", "RunsRaggedArray", "get_pileup", "get_boolean_mask", "merge_intervals"]
