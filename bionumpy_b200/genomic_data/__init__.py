"""Genomes and data on them (bionumpy/genomic_data), for in-memory intervals and tracks."""
from .genome import Genome, GenomicIntervals, GenomicArray, ignore_underscores, keep_all

__all__ = ["Genome", "GenomicIntervals", "GenomicArray", "ignore_underscores", "keep_all"]
