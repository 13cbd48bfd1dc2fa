"""Interval arithmetics on the device (bionumpy/arithmetics): pileups, masks and merges of the intervals of one
contig, operators between run-length tracks, intersections, sorting and similarity of interval sets."""
from .intervals import (FloatRunLengthArray, GenomicRunLengthArray, RunsRaggedArray, count_overlap, get_boolean_mask, get_pileup,
                        global_intersect, intersect, merge_intervals, sort_intervals, unique_intersect)
from .similarity_measures import forbes, get_contingency_table, jaccard

__all__ = ["FloatRunLengthArray", "GenomicRunLengthArray", "RunsRaggedArray", "get_pileup", "get_boolean_mask", "merge_intervals",
           "count_overlap", "intersect", "global_intersect", "unique_intersect", "sort_intervals", "forbes", "jaccard",
           "get_contingency_table"]
