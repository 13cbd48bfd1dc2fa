"""bionumpy_b200 -- an H100-native (sm_90a) k-mer hot path behind BioNumPy's API names.

    import bionumpy_b200 as bnp
    for chunk in bnp.open("reads.fq.gz").read_chunks():
        kmers = bnp.get_kmers(chunk.sequence, 31)            # lazy
        hist += bnp.count_hashed(kmers, 1 << 24)             # fused hash + histogram on the GPU

Only the ragged-sequence path is implemented (see DESIGN.md): FASTQ/FASTA chunk bytes -> row
offsets -> 2-bit codes -> rolling k-mer hash -> [sliding-window minimizer] -> bincount.  All
compute runs in libbnpk.so (hand-written CUDA, C-ABI in include/bnpk.h); there is no CPU fallback.
"""
from . import config
from .encoded_array import (EncodedArray, EncodedRaggedArray, as_encoded_array, change_encoding, BaseEncoding,
                            from_encoded_array, EncodingException)
from .ragged import RaggedArray, RaggedShape
from .encodings import (AlphabetEncoding, DNAEncoding, ACTGEncoding, ACGTEncoding, KmerEncoding, EncodingError,
                        AminoAcidEncoding, RNAENcoding, StrandEncoding)
from . import encodings, sequence, io, streams
from .sequence import (get_kmers, get_minimizers, count_encoded, count_kmers, count_hashed, count_kmers_hashed,
                       EncodedCounts, complement, get_reverse_complement, get_motif_scores, match_string)
from .streams import streamable, bincount, BnpStream
from .io import bnp_open, FormatException, IndexedFasta, open_indexed
from .sequence import KmerIndex, KmerLookup, BloomFilter
from .sequence import count_kmers_exact, KmerCounter, KmerCounts
from .io.buffers import CudaFastQBuffer, CudaTwoLineFastaBuffer, FastQBuffer, TwoLineFastaBuffer
from .io.multiline import CudaMultiLineFastaBuffer, MultiLineFastaBuffer
from .datatypes import (SequenceEntry, SequenceEntryWithQuality, Interval, StrandedInterval, Bed6, BedGraph, BamEntry,
                        replace)
from . import datatypes
from . import arithmetics, genomic_data, alignments
from .genomic_data import Genome, GenomicIntervals, GenomicArray
from .io.files import count_entries
from .io.write import NpBufferedWriter

open = bnp_open

__version__ = "0.1.0"
