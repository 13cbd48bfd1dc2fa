from .buffers import (CudaFastQBuffer, CudaTwoLineFastaBuffer, CudaOneLineBuffer, FastQBuffer, TwoLineFastaBuffer,
                      FieldView)
from .exceptions import FormatException, IncompleteEntryException
from .files import bnp_open, count_entries
from .bgzf import BgzfWriter
from .write import NpBufferedWriter
from .parser import CudaFileReader, NpDataclassReader
from .multiline import CudaMultiLineFastaBuffer, MultiLineFastaBuffer
from .indexed_fasta import IndexedFasta, read_index, create_index, open_indexed
from .delimited import DelimitedBuffer, BedBuffer, Bed6Buffer, BdgBuffer, BedGraphBuffer, GTFBuffer, GFFBuffer, \
    NarrowPeakBuffer
from .motifs import read_motif
from .bam import BamBuffer, BamIntervalBuffer
from .sam import SAMBuffer, SAMIntervalBuffer
from . import bam, sam
