"""Genomes and data on them (bionumpy/genomic_data), for in-memory intervals and tracks."""
from .genome import (Genome, GenomicIntervals, GenomicLocation, GenomicArray, GenomicAnnotation, Genes, Transcripts, Exons,
                     ignore_underscores, keep_all)

__all__ = ["Genome", "GenomicIntervals", "GenomicLocation", "GenomicArray", "GenomicAnnotation", "Genes", "Transcripts", "Exons",
           "ignore_underscores", "keep_all"]
