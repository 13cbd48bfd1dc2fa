from ..encoded_array import BaseEncoding, Encoding, OneToOneEncoding, ASCIIEncoding
from .alphabet_encoding import (AlphabetEncoding, ACTGEncoding, ACGTEncoding, DNAEncoding, ACUGEncoding,
                                RNAENcoding, AminoAcidEncoding, StrandEncoding, BamEncoding,
                                CigarOpEncoding)
from .kmer_encodings import KmerEncoding
from .exceptions import EncodingError
