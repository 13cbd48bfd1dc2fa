from .kmers import get_kmers, count_kmers, count_kmers_hashed
from .exact_counts import count_kmers_exact, KmerCounter, KmerCounts
from .minimizers import get_minimizers
from .count_encoded import count_encoded, count_hashed, EncodedCounts
from .dna import complement, get_reverse_complement, get_sequences, get_strand_specific_sequences
from .indexing import KmerIndex, KmerLookup
from .bloom_filter import BloomFilter
from .position_weight_matrix import get_motif_scores, PWM
from .string_matcher import match_string, StringMatcher, FixedLenRegexMatcher, RegexMatcher
