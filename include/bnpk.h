/*
 * bnpk.h -- C-ABI of libbnpk.so, the H100 (sm_90a) k-mer hot path behind BioNumPy's API.
 *
 * This is the drop-in boundary: plain pointers and sizes, no torch types.  The reference
 * (bionumpy @ 6773266) is pure Python/NumPy and has no FFI; the seam it offers for this path
 * is `bnp.set_backend(lib)` + `CupyFileReader` (bionumpy/__init__.py:47-94,
 * bionumpy/cupy_compatible/parser.py:10-17) and the `buffer_type=` plug-in protocol
 * (bionumpy/io/files.py:52-68, bionumpy/io/file_buffers.py:80-271).  Each entry point below
 * names the reference function(s) it replaces (paths relative to /root/reference/bionumpy/).
 * INTEGRATION.md shows the ctypes stub a reference maintainer would add.
 *
 * Conventions
 *   - every pointer is a DEVICE pointer unless its name ends in `_host`;
 *   - `stream` is a cudaStream_t passed as void* (NULL = legacy default stream);
 *   - all work is stream-ordered and asynchronous; nothing here synchronises unless stated;
 *   - inputs are borrowed and never written; outputs are caller-allocated;
 *   - return value: 0 = ok, >0 = cudaError_t, <0 = BNPK_E_* argument error;
 *     `bnpk_last_error()` gives a thread-local message;
 *   - kernels never trap on bad data: they fill a device-side `bnpk_status` block that the
 *     host reads when it chooses to (the Python layer turns it into the reference's
 *     FormatException(line_number) / EncodingError(offset)).
 */
#ifndef BNPK_H
#define BNPK_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define BNPK_ABI_VERSION 3

/* argument errors */
#define BNPK_E_BADARG   (-1)
#define BNPK_E_K        (-2)   /* k outside 1..31            (sequence/kmers.py:69)        */
#define BNPK_E_WINDOW   (-3)   /* window_size < k            (sequence/minimizers.py:50)   */
#define BNPK_E_WORKSPACE (-4)  /* workspace too small                                      */
#define BNPK_E_BINS     (-5)

/* byte -> 2-bit code modes (encodings/alphabet_encoding.py:19-46,102-107).  Modes 0-2 are
 * closed-form bit tricks; mode 3 uses a caller-supplied 256-byte LUT (any 4-letter alphabet,
 * e.g. RNA "ACUG"; 255 = invalid), which is what AlphabetEncoding._lookup is. */
#define BNPK_ENC_ASCII_ACGT 0  /* DNAEncoding  A/a0 C/c1 G/g2 T/t3                        */
#define BNPK_ENC_ASCII_ACTG 1  /* ACTGEncoding A/a0 C/c1 T/t2 G/g3                        */
#define BNPK_ENC_CODES      2  /* bytes already are codes 0..3 (an encoded EncodedArray)  */
#define BNPK_ENC_LUT        3

/* histogram modes */
#define BNPK_HIST_AUTO   0     /* smem-privatised when bins fit, else global atomics       */
#define BNPK_HIST_SMEM   1
#define BNPK_HIST_GLOBAL 2

/* Device-side status block (int64[16]); zero/sentinel-initialised by bnpk_status_init. */
enum {
    BNPK_ST_N_LINES = 0,       /* newlines seen in the chunk                               */
    BNPK_ST_N_RECORDS = 1,     /* complete entries = n_lines / lines_per_entry             */
    BNPK_ST_N_COMPLETE_BYTES = 2, /* bytes up to and including the last kept newline
                                     (FileBuffer.size, io/one_line_buffer.py:67-69)        */
    BNPK_ST_BAD_HEADER_ENTRY = 3, /* min entry whose first byte != header char (INT64_MAX = none)
                                     -> FormatException(line_number = entry*lines_per_entry),
                                     io/one_line_buffer.py:155-173                         */
    BNPK_ST_BAD_PLUS_ENTRY = 4,   /* min entry whose 3rd line does not start with '+'
                                     -> line_number = 2 + entry*4, io/fastq_buffer.py:38-45 */
    BNPK_ST_BAD_BASE = 5,      /* min (row << 32 | position-in-row) of a byte outside the
                                  alphabet (INT64_MAX = none) -> EncodingError(offset),
                                  encodings/alphabet_encoding.py:34-46                     */
    BNPK_ST_N_BASES = 6,       /* sum of row lengths processed                             */
    BNPK_ST_N_VALUES = 7,      /* k-mers / minimizers produced or counted                  */
    BNPK_ST_N_LONG_ROWS = 8,   /* rows that did not fit a tile halo and took the long path */
    BNPK_ST_CR = 9,            /* 1 if '\r' trimming is active (io/one_line_buffer.py:175-182) */
    BNPK_ST_LAST_ROW_START = 10, /* internal: 1 + start of the last sequence line counted  */
    BNPK_ST_LAST_ROW_INDEX = 11, /* internal: 1 + its entry index                          */
    BNPK_ST_OVERFLOW = 12,     /* != 0: the fused pass met more long/odd rows than its scratch holds;
                                  the counts are incomplete -- use bnpk_line_split + bnpk_rows_kmer_count */
    BNPK_ST_TABLE_FULL = 13,   /* != 0: a k-mer table insert probed every slot without finding room; the table misses
                                  k-mers.  Callers that keep the table at most half full never see it */
    BNPK_ST_WORDS = 16
};

int         bnpk_abi_version(void);
const char *bnpk_last_error(void);
/* number of SMs of the current device, for callers that size their own grids */
int         bnpk_sm_count(void);

/* Initialise a status block (device int64[BNPK_ST_WORDS]). */
int bnpk_status_init(int64_t *status, void *stream);

/* ---------------------------------------------------------------------------------------
 * K0  byte census.  Replaces nothing by itself; lets a caller size the outputs of
 *     bnpk_line_split exactly (the reference gets the size from np.flatnonzero's result,
 *     io/one_line_buffer.py:63).  count_out: device int64[1].
 * ------------------------------------------------------------------------------------- */
int bnpk_count_byte(const uint8_t *chunk, size_t n, uint8_t value, int64_t *count_out, void *stream);

/* ---------------------------------------------------------------------------------------
 * K1  line split.  Replaces OneLineBuffer.from_raw_buffer + _validate +
 *     _get_buffer_extractor (io/one_line_buffer.py:44-71,139-173), FastQBuffer._validate
 *     (io/fastq_buffer.py:38-45) and TextBufferExtractor.get_field_by_number
 *     (io/file_buffers.py:315-338) for ONE field of every complete entry.
 *
 *   lines_per_entry  4 (FASTQ) or 2 (two-line FASTA)
 *   field_line       which line of the entry (FASTQ: 0 name, 1 sequence, 3 quality)
 *   start_offset     bytes skipped at the line start (_line_offsets: 1 for the header line)
 *   header_char      '@' or '>';  check_plus: validate the '+' line (FASTQ)
 *   trim_cr          -1 = decide like the reference (first entries' header ends in '\r'),
 *                    0 = never, 1 = always
 *   starts/lens      out, capacity `max_rows` rows (extra rows are counted, not written)
 *   status           device int64[BNPK_ST_WORDS], pre-initialised
 *   workspace        device scratch of bnpk_tile_workspace_bytes(n) bytes (look-back state, deferred
 *                    long-row list and a 64 MiB table of 32-bit counters used by K6 for global
 *                    tables of 2^22..2^24 bins).  The entry points clear what they use on the first
 *                    slice of a chunk; bnpk_tile_workspace_reset zeroes all of it.
 * A single pass over the chunk (decoupled look-back over per-tile newline counts).
 * ------------------------------------------------------------------------------------- */
size_t bnpk_tile_workspace_bytes(size_t n);
int    bnpk_tile_workspace_reset(void *workspace, size_t workspace_bytes, void *stream);
int bnpk_line_split(const uint8_t *chunk, size_t n, int lines_per_entry, int field_line,
                    int start_offset, uint8_t header_char, int check_plus, int trim_cr,
                    int64_t *starts, int32_t *lens, size_t max_rows,
                    int64_t *status, void *workspace, size_t workspace_bytes, void *stream);

/* ---------------------------------------------------------------------------------------
 * K6  fused count: raw FASTQ / two-line FASTA chunk bytes -> histogram, never materialising
 *     offsets, codes or hashes.  Replaces, for one chunk, the chain
 *       OneLineBuffer.from_raw_buffer            io/one_line_buffer.py:44-71
 *       change_encoding(..., DNAEncoding)        encoded_array.py:655-695 -> alphabet_encoding.py:34-46
 *       _get_dna_kmers                           sequence/kmers.py:105-126
 *       [get_minimizers]                         sequence/minimizers.py:20-54
 *       count_encoded(axis=None)                 sequence/count_encoded.py:150-188
 *     hist[b] += #{values v : v mod n_bins == b} over all COMPLETE entries of the chunk
 *     (n_bins = 4^k gives the reference's exact np.bincount; other n_bins = the hashed-bucket
 *     extension).  window_size = 0 counts k-mers, otherwise minimizers (window in bases).
 *     hist is int64[n_bins] and is ACCUMULATED into (zero it yourself for a fresh count).
 *     Chunks may be fed in slices: call with the same workspace/status and consecutive
 *     [slice_begin, slice_end) byte ranges of one resident buffer; `final` marks the last.
 *     Residency: a non-final call reads only chunk[0, slice_end), so the bytes from slice_end
 *     on may still be in flight (the host pipeline copies slice s+1 while slice s is counted);
 *     the final call may read all n bytes.  Empty slices and an empty final slice [n, n) are
 *     allowed.  A call counts the 16 KiB tiles whose bytes and 2 KiB halo are resident, so
 *     calls that end before byte 18432 (and are not final) count nothing.
 *     '\r' trimming (trim_cr = -1) is decided by the call that counts the first tile, from all
 *     bytes resident then: at least 18 KiB, or the whole chunk.  A sliced count can therefore
 *     differ from a one-shot launch only if the first header line lacks '\r', a later one of
 *     the first lines_per_entry headers ends in '\r', and those headers do not all lie in the
 *     bytes resident at that call.
 * ------------------------------------------------------------------------------------- */
int bnpk_chunk_kmer_count(const uint8_t *chunk, size_t n, size_t slice_begin, size_t slice_end,
                          int final_slice, int lines_per_entry, uint8_t header_char, int check_plus,
                          int trim_cr, int enc_mode, const uint8_t *lut256, int k, int window_size,
                          int64_t n_bins, int hist_mode, int64_t *hist,
                          int64_t *status, void *workspace, size_t workspace_bytes, void *stream);

/* ---------------------------------------------------------------------------------------
 * Row-driven kernels: operate on an arbitrary ragged view (base bytes, starts[R], lens[R])
 * -- what EncodedRaggedArray(data, RaggedView2(starts, lens)) is (io/file_buffers.py:335-338).
 * `offsets` are int64[R+1] exclusive prefix sums produced by bnpk_row_offsets.
 * ------------------------------------------------------------------------------------- */

/* offsets[r] = sum_{q<r} max(lens[q] - shrink, 0); offsets[R] = total.  (The ragged shape of
 * out[..., :-shrink], sequence/kmers.py:100, sequence/rollable.py:66.)  workspace as for K1
 * with n := R. */
int bnpk_row_offsets(const int32_t *lens, size_t n_rows, int shrink, int64_t *offsets,
                     void *workspace, size_t workspace_bytes, void *stream);

/* K2  change_encoding / AlphabetEncoding._encode (encoded_array.py:655-695,
 *     alphabet_encoding.py:34-46): gather the rows contiguously and map bytes to codes. */
int bnpk_rows_encode(const uint8_t *base, size_t base_bytes, const int64_t *starts, const int32_t *lens, size_t n_rows,
                     int enc_mode, const uint8_t *lut256, const int64_t *offsets, uint8_t *codes_out,
                     int64_t *status, void *stream);

/* K3  get_kmers / _get_dna_kmers + the ragged [..., :-k+1] (sequence/kmers.py:36-126):
 *     out[offsets[r] + i] = sum_j code[r][i+j] * 4^j  (int64), offsets from shrink = k-1. */
int bnpk_rows_kmer_hash(const uint8_t *base, size_t base_bytes, const int64_t *starts, const int32_t *lens, size_t n_rows,
                        int enc_mode, const uint8_t *lut256, int k, const int64_t *offsets,
                        int64_t *hashes_out, int64_t *status, void *stream);

/* K3' the reference's generic path for alphabets whose size is not 4 (KmerEncoder dot product,
 *     sequence/kmers.py:17-27,87): out[offsets[r] + i] = sum_j code[r][i+j] * alphabet_size^j in
 *     int64 (wrapping) arithmetic.  lut256 maps bytes to codes (255 = invalid), NULL = bytes are codes. */
int bnpk_rows_generic_hash(const uint8_t *base, size_t base_bytes, const int64_t *starts, const int32_t *lens, size_t n_rows,
                           const uint8_t *lut256, int alphabet_size, int k, const int64_t *offsets,
                           int64_t *hashes_out, int64_t *status, void *stream);

/* K4  get_minimizers (sequence/minimizers.py:20-54): out[offsets[r] + j] = min of the
 *     window_size-k+1 k-mer hashes of window j; offsets from shrink = window_size-1. */
int bnpk_rows_minimizers(const uint8_t *base, size_t base_bytes, const int64_t *starts, const int32_t *lens, size_t n_rows,
                         int enc_mode, const uint8_t *lut256, int k, int window_size,
                         const int64_t *offsets, int64_t *mins_out, int64_t *status, void *stream);

/* K3+K5 / K4+K5 fused on a ragged view: get_kmers|get_minimizers -> count_encoded(axis=None)
 *     without materialising the values (sequence/kmers.py:129-145 count_kmers). */
int bnpk_rows_kmer_count(const uint8_t *base, size_t base_bytes, const int64_t *starts, const int32_t *lens, size_t n_rows,
                         int enc_mode, const uint8_t *lut256, int k, int window_size,
                         int64_t n_bins, int hist_mode, int64_t *hist, int64_t *status, void *stream);

/* get_reverse_complement (sequence/dna.py:36-65: complement Lookup, then every row reversed):
 *     out[offsets[r] + i] = lut256[base[starts[r] + lens[r] - 1 - i]]; offsets from shrink = 0.  lut256 (device) is
 *     the complement table of the array's encoding (_get_complement_lookup, sequence/dna.py:13-34). */
int bnpk_rows_reverse_complement(const uint8_t *base, size_t base_bytes, const int64_t *starts, const int32_t *lens,
                                 size_t n_rows, const uint8_t *lut256, const int64_t *offsets, uint8_t *out, void *stream);

/* EXTENSION (no reference counterpart; what Jellyfish --canonical does, benchmarks/rules/kmer_counting.smk:11):
 *     canonical k-mers = min(h, hash of the reverse complement of the same k-mer).  complement_xor is the
 *     complement as an XOR on a 2-bit code: 3 for "ACGT"-ordered alphabets (DNAEncoding), 2 for "ACTG"-ordered.
 *     Same outputs as bnpk_rows_kmer_hash / bnpk_rows_kmer_count otherwise. */
int bnpk_rows_kmer_hash_canonical(const uint8_t *base, size_t base_bytes, const int64_t *starts, const int32_t *lens,
                                  size_t n_rows, int enc_mode, const uint8_t *lut256, int k, int complement_xor,
                                  const int64_t *offsets, int64_t *hashes_out, int64_t *status, void *stream);
int bnpk_rows_kmer_count_canonical(const uint8_t *base, size_t base_bytes, const int64_t *starts, const int32_t *lens,
                                   size_t n_rows, int enc_mode, const uint8_t *lut256, int k, int complement_xor,
                                   int64_t n_bins, int hist_mode, int64_t *hist, int64_t *status, void *stream);

/* EXTENSION (no reference counterpart; what `jellyfish count` produces, benchmarks/rules/kmer_counting.smk:1-31): exact
 *     counts of distinct k-mers, any k in 1..31, in an open-addressing hash table in device memory.
 *     Table = keys int64[capacity] + counts int64[capacity], capacity a power of two; a free slot has key -1 and count 0
 *     (clear a table by filling keys with -1 and counts with 0).  Key = the k-mer hash of bnpk_rows_kmer_hash (with
 *     complement_xor 1..3: the canonical hash of bnpk_rows_kmer_hash_canonical; 0 = forward k-mers); its home slot is
 *     splitmix64(key) mod capacity, collisions probe linearly.  The k-mers of every row are inserted (count + 1 each);
 *     *n_used (device int64) is increased by the number of slots this call claimed.  The caller keeps the table at most
 *     half full (n_used + positions of the call <= capacity / 2), so an insert always finds room; if it does not, the
 *     k-mer is dropped and status[BNPK_ST_TABLE_FULL] is set.  Bad bases are reported as by bnpk_rows_kmer_hash, but the
 *     row's k-mers are still inserted.  BNPK_E_BADARG for a capacity that is not a power of two, BNPK_E_K for k
 *     outside 1..31. */
int bnpk_rows_kmer_table_insert(const uint8_t *base, size_t base_bytes, const int64_t *starts, const int32_t *lens,
                                size_t n_rows, int enc_mode, const uint8_t *lut256, int k, int complement_xor,
                                int64_t *keys, int64_t *counts, size_t capacity, int64_t *n_used,
                                int64_t *status, void *stream);
/*     Growth: every (key, count) of a table is inserted into a second (cleared, larger) table with the same slot function;
 *     *n_used is increased by the slots claimed there.  Both capacities must be powers of two. */
int bnpk_kmer_table_rehash(const int64_t *keys, const int64_t *counts, size_t capacity,
                           int64_t *new_keys, int64_t *new_counts, size_t new_capacity, int64_t *n_used,
                           int64_t *status, void *stream);

/* K7  motif scores of a position weight matrix: get_motif_scores / PWM.calculate_scores
 *     (sequence/position_weight_matrix.py:83-100,166-196).  matrix[j * alphabet_size + c] (device float64) is the
 *     score of code c at motif column j, the transpose of the reference's PWM._matrix[c, j]; motif_len = m.
 *     out[offsets[r] + i] = ((+0.0 + matrix[0][code[r][i]]) + matrix[1][code[r][i+1]]) + ... summed in column order in
 *     float64, which is the reference's sequence of adds, so the bits are the reference's.  tail = 0: the windows of
 *     the row, max(L - m + 1, 0) values (offsets from shrink = m - 1; the reference's [..., :-m+1]); tail = 1: also the
 *     last m - 1 positions with the columns that fit, L values (shrink = 0; calculate_scores on one flat row).
 *     Text is read as by the other row entry points (enc_mode, lut256: AlphabetEncoding(pwm.alphabet)); for an
 *     alphabet_size that is not 4 only BNPK_ENC_LUT (lut256: byte -> code, 255 = invalid) and BNPK_ENC_CODES (bytes
 *     are codes, valid below alphabet_size) are accepted.  A byte outside the alphabet anywhere in a row, including its
 *     last m - 1 bytes, is reported in status[BNPK_ST_BAD_BASE] (EncodingError, encodings/alphabet_encoding.py:34-46);
 *     N_BASES += row lengths, N_VALUES += values scored.  BNPK_E_BADARG unless 1 <= motif_len <= 1024,
 *     2 <= alphabet_size <= 255 and alphabet_size * motif_len <= 8192 (the table lives in shared memory). */
int bnpk_rows_pwm_scores(const uint8_t *base, size_t base_bytes, const int64_t *starts, const int32_t *lens,
                         size_t n_rows, int enc_mode, const uint8_t *lut256, int alphabet_size,
                         const double *matrix /* [m][alphabet_size] */, int motif_len, int tail,
                         const int64_t *offsets, double *scores_out, int64_t *status, void *stream);
/*     get_motif_scores(...).max(axis=-1) without writing the scores: max_out[r] = the largest score of row r's windows
 *     (tail = 0), NaN if one of them is NaN (np.max), -inf for a row without a window.  Same arguments and status. */
int bnpk_rows_pwm_max(const uint8_t *base, size_t base_bytes, const int64_t *starts, const int32_t *lens,
                      size_t n_rows, int enc_mode, const uint8_t *lut256, int alphabet_size,
                      const double *matrix, int motif_len, double *max_out, int64_t *status, void *stream);

/* K8  string and pattern matches: match_string, StringMatcher, FixedLenRegexMatcher, RegexMatcher
 *     (sequence/string_matcher.py).  A pattern is n_sub sub-patterns (one per combination of gap lengths; 1..64) of
 *     sub_lens[k] columns each (host int32; 1..1024).  Their columns, concatenated in order, are symbol sets in
 *     `sets` (device): column c is the words sets[c * W .. c * W + W - 1], W = ceil(alphabet_size / 32), and code s
 *     matches there iff bit s % 32 of word s / 32 is set.  match_out[offsets[r] + p] = 1 iff some sub-pattern matches
 *     at position p of row r and fits inside the row, else 0.  same = 0: the positions of the longest sub-pattern's
 *     windows, max(L - span + 1, 0) per row (span = the longest sub-pattern; offsets from shrink = span - 1);
 *     same = 1: every position, L per row (shrink = 0).
 *     Text is read as by the other row entry points (enc_mode, lut256); an alphabet_size that is not 4 takes
 *     BNPK_ENC_LUT (lut256: byte -> code, 255 = invalid) or BNPK_ENC_CODES (bytes are codes, valid below
 *     alphabet_size), and alphabet_size 256 means raw bytes: BNPK_ENC_CODES, every byte valid and its own code.
 *     A byte outside the alphabet anywhere in a row is reported in status[BNPK_ST_BAD_BASE]; N_BASES += row lengths,
 *     N_VALUES += positions tested.  BNPK_E_BADARG unless 2 <= alphabet_size <= 256, the sub-pattern limits above
 *     hold and the sets fit 8192 words (32 KiB of shared memory: total columns * W <= 8192). */
int bnpk_rows_match(const uint8_t *base, size_t base_bytes, const int64_t *starts, const int32_t *lens, size_t n_rows,
                    int enc_mode, const uint8_t *lut256, int alphabet_size, const uint32_t *sets,
                    const int32_t *sub_lens, int n_sub, int same, const int64_t *offsets, uint8_t *match_out,
                    int64_t *status, void *stream);
/*     The matches of every row counted without writing them: count_out[r] (int64) = the number of ones row r's
 *     match_out would hold.  Same arguments and status. */
int bnpk_rows_match_count(const uint8_t *base, size_t base_bytes, const int64_t *starts, const int32_t *lens,
                          size_t n_rows, int enc_mode, const uint8_t *lut256, int alphabet_size, const uint32_t *sets,
                          const int32_t *sub_lens, int n_sub, int same, int64_t *count_out, int64_t *status,
                          void *stream);

/* K5  np.bincount(values % n_bins, minlength=n_bins) accumulated into hist
 *     (sequence/count_encoded.py:173-177; EncodedArray.__array_function__ encoded_array.py:459-460).
 *     Values must be non-negative; n_bins = len(alphabet) reproduces count_encoded exactly
 *     (out-of-range values are reported in status[BNPK_ST_BAD_BASE]). */
int bnpk_bincount(const int64_t *values, size_t n, int64_t n_bins, int hist_mode, int64_t *hist,
                  int64_t *status, void *stream);

/* K5' count_encoded(axis=-1) (sequence/count_encoded.py:180-182): per-row bincount,
 *     out[r * n_bins + b]; offsets int64[R+1] delimit the rows of `values`. */
int bnpk_bincount_rows(const int64_t *values, const int64_t *offsets, size_t n_rows, int64_t n_bins,
                       int64_t *out, int64_t *status, void *stream);

/* Multi-line FASTA bookkeeping over the per-line arrays of bnpk_line_split(lines_per_entry = 1)
 * (MultiLineFastaBuffer.from_raw_buffer / get_data, io/multiline_buffer.py:46-62,89-106):
 *   bnpk_multiline_flags    is_header[i] (line starts with '>'), out2[0] = 1 + the last line whose newline is followed by
 *                           '>' (0: no complete entry), out2[1] = 1 if one of the first ten lines ends in '\r'
 *   bnpk_multiline_entries  with hdr_before = bnpk_row_offsets(is_header, 0): header fields (h_starts/h_lens per entry),
 *                           the sequence lines compacted in order (s_starts/s_lens) and entry_lens (zero-initialised by
 *                           the caller) = bases per entry; trim_cr as decided from out2[1]. */
int bnpk_multiline_flags(const uint8_t *chunk, size_t n, const int64_t *line_starts, const int32_t *line_lens, size_t n_lines,
                         int32_t *is_header, int64_t *out2, void *stream);
int bnpk_multiline_entries(const uint8_t *chunk, const int64_t *line_starts, const int32_t *line_lens, const int32_t *is_header,
                           const int64_t *hdr_before, size_t keep, int trim_cr, int64_t *h_starts, int32_t *h_lens,
                           int64_t *s_starts, int32_t *s_lens, int64_t *entry_lens, void *stream);

/* ---------------------------------------------------------------------------------------
 * Intervals (BED; io/delimited_buffers.py:29-316, io/indexed_fasta.py:165-206, sequence/dna.py:68-106).
 *
 * bnpk_delimited_columns: the tab-separated columns of every line of a chunk, over the per-line arrays of
 *   bnpk_line_split(lines_per_entry = 1).  The column count is the first line's; `columns` is a HOST array of n_columns
 *   bnpk_column (n_columns <= BNPK_MAX_COLUMNS), column c of every line is written as its kind says:
 *     BNPK_COL_SKIP        nothing (the column is still counted)
 *     BNPK_COL_TEXT        out = int64[n_lines] chunk offset of the field, lens = int32[n_lines] its length
 *     BNPK_COL_INT         out = int64[n_lines]: an optional '-' or '+' and 1 to 18 digits
 *     BNPK_COL_INT_OR_DOT  as BNPK_COL_INT, and "." reads as 0 (Optional[int], io/strops.py:69-83)
 *     BNPK_COL_STRAND      out = uint8[n_lines] StrandEncoding code: '+' 0, '-' 1, '.' 2
 *   When the first line ends in '\r', a '\r' that ends a line is not part of its last column.  The first fault is
 *   atomicMin-ed into status[BNPK_ST_BAD_BASE] as (line << 8 | column << 3 | BNPK_BAD_*) (status pre-initialised).
 *   BNPK_E_BADARG for a NULL pointer with n_lines > 0, n_columns outside 1..BNPK_MAX_COLUMNS, an unknown kind or a
 *   missing output.
 * bnpk_name_lookup: out_ids[r] = the index k of the name table with names[name_offsets[k] .. name_offsets[k + 1]) equal
 *   to the bytes of row r (base[starts[r] .. + lens[r])), compared byte for byte over their full lengths.  The table
 *   must be sorted as bytes (a name before every longer name it is a prefix of).  A row with no name gets -1 and is
 *   atomicMin-ed into status[BNPK_ST_BAD_BASE].
 * bnpk_interval_gather: row r = bases [start[r], stop[r]) of contig ids[r], whose first base is file byte
 *   contig_offset[id] (.fai column 3), with lenc[id] bases per line of lenb[id] bytes (.fai columns 4, 5), contig_len[id]
 *   bases, line ends skipped; IndexedFasta.__getitem__ (io/indexed_fasta.py:101-131) is the consecutive rows that cover
 *   [0, contig_len[id]), get_interval_sequences any rows.  ids == NULL is the flat
 *   mode: one contig of file_bytes bases, no line ends (contig_* are not read).  A row with start < 0, stop < start,
 *   stop > the contig length, more than INT32_MAX bases, a contig id outside 0..n_contigs-1 or a base outside the file is atomicMin-ed into
 *   status[BNPK_ST_BAD_BASE].  Two passes:
 *     out == NULL   check pass: row_lens[r] = stop - start for a good row, 0 for a reported one
 *     out != NULL   copy pass: out[out_offsets[r] + i], out_offsets int64[R+1] of the check pass' row_lens; a row whose
 *                   strand[r] != 0 (strand may be NULL) is written reverse-complemented through complement_lut256.
 * ------------------------------------------------------------------------------------- */
#define BNPK_MAX_COLUMNS 16
#define BNPK_COL_SKIP        0
#define BNPK_COL_TEXT        1
#define BNPK_COL_INT         2
#define BNPK_COL_INT_OR_DOT  3
#define BNPK_COL_STRAND      4
#define BNPK_BAD_TABS        1   /* the line's tab count differs from the first line's      */
#define BNPK_BAD_COLUMNS     2   /* the line has fewer columns than `columns` names         */
#define BNPK_BAD_INT         3   /* not an integer of at most 18 digits                     */
#define BNPK_BAD_STRAND      4   /* not one of '+', '-', '.'                                */

typedef struct bnpk_column {
    int kind;
    void *out;
    int32_t *lens;
} bnpk_column;

int bnpk_delimited_columns(const uint8_t *chunk, size_t n, const int64_t *line_starts, const int32_t *line_lens,
                           size_t n_lines, const bnpk_column *columns, int n_columns, int64_t *status, void *stream);
int bnpk_name_lookup(const uint8_t *base, size_t base_bytes, const int64_t *starts, const int32_t *lens, size_t n_rows,
                     const uint8_t *names, const int64_t *name_offsets, size_t n_names, int32_t *out_ids,
                     int64_t *status, void *stream);
int bnpk_interval_gather(const uint8_t *file, size_t file_bytes, size_t n_rows, const int32_t *ids,
                         const int64_t *contig_offset, const int32_t *lenc, const int32_t *lenb, const int64_t *contig_len,
                         size_t n_contigs, const int64_t *start, const int64_t *stop, const uint8_t *strand,
                         const uint8_t *complement_lut256, int32_t *row_lens, const int64_t *out_offsets, uint8_t *out,
                         int64_t *status, void *stream);

/* ---------------------------------------------------------------------------------------
 * Pileups, run-length tracks and interval merges (get_pileup, get_boolean_mask, merge_intervals
 * arithmetics/intervals.py:137-304; GenomicRunLengthArray and GenomicArray, genomic_data/genomic_track.py).
 * Positions are int64 in [0, 2^59).  A track of size S is R runs: run_starts int64[R + 1] (run_starts[0] = 0,
 * increasing, run_starts[R] = S) and values int64[R]; no two neighbouring runs have the same value.
 *
 * bnpk_interval_events: row r = [start[r], stop[r]) of contig ids[r] (contig_offset[id] is its first global position,
 *   contig_len[id] its size; a contig with contig_offset < 0 is left out: its rows are not checked and become empty
 *   intervals at 0).  ids == NULL: every row is on one contig [0, size).  A row with start < 0, stop < start,
 *   stop > the contig size or an id outside 0..n_contigs-1 is atomicMin-ed into status[BNPK_ST_BAD_BASE] and becomes
 *   an empty interval at 0.  keys int64[2R] (may be NULL): keys[2r] = global start << 1 | 1, keys[2r + 1] = global
 *   stop << 1; g_start / g_stop int64[R] (may be NULL): the global start and stop.
 * bnpk_pileup_runs: the runs of the coverage of the intervals whose event keys (bnpk_interval_events) are sorted in
 *   keys[0 .. n_keys): BNPK_PILEUP_COUNT the number of intervals over each position, BNPK_PILEUP_ANY 1 where there is
 *   at least one and 0 elsewhere.  Writes *n_runs = R (<= n_keys + 1), run_starts[0 .. R] (capacity n_keys + 2) and
 *   run_values[0 .. R) (capacity n_keys + 1).  Keys at positions >= size add nothing.  workspace as for
 *   bnpk_row_offsets with n := n_keys (2 look-back words per 2048 keys).
 * bnpk_runs_reduce: out[q] = the reduction over positions [q_start[q], q_stop[q]) (clipped to [0, S)) of the track:
 *   BNPK_RUNS_MAX / BNPK_RUNS_MIN the largest / smallest value, BNPK_RUNS_SUM the sum of value x positions (int64,
 *   wrapping), BNPK_RUNS_ANY 1 if a value is not 0.  An empty query gives INT64_MIN, INT64_MAX, 0 and 0.  scratch
 *   is device int64[3 * n_q + 1]; workspace as for bnpk_row_offsets with n := n_q.  No synchronisation.
 * bnpk_runs_extract: out[out_offsets[q] + i] = the value at position q_start[q] + i, for i < out_offsets[q + 1] -
 *   out_offsets[q]; every such position must lie in [0, S).
 * bnpk_interval_merge: merge_intervals (arithmetics/intervals.py:270-304) over rows sorted by start inside each
 *   segment; a segment is a maximal block of rows whose same_prev[r] != 0 (row r continues row r - 1's segment;
 *   same_prev NULL: one segment).  stops = the running max of stop in the segment; row r starts a group iff it starts
 *   a segment or start[r] > stops[r - 1] + distance.  out_rows[g] = the first row of group g, out_stops[g] = the
 *   group's largest stop, *n_out = the number of groups.  A row whose start is smaller than the previous row's in the
 *   same segment is atomicMin-ed into status[BNPK_ST_BAD_BASE].  workspace as for bnpk_row_offsets with n := n_rows.
 * bnpk_rows_equal_prev: flag[r] = 1 iff r > 0 and the bytes of row r equal those of row r - 1 (same length, every
 *   byte), else 0.
 * bnpk_runs_combine: op(A, B) of two tracks of one size S (a_starts[n_a] == b_starts[n_b] == S, checked by the caller)
 *   whose runs are non-empty but whose neighbouring runs may have equal values.  P is the union of both tracks' run
 *   starts; the value on [p, the next point of P) is op(A(p), B(p)) in int64, and a run starts at p where p == 0 or
 *   the value differs from the value at the previous point of P, so the output is canonical.  Writes *n_out = R
 *   (<= n_a + n_b), out_starts[0 .. R] (capacity n_a + n_b + 1, out_starts[R] = S) and out_values[0 .. R).  BNPK_OP_ADD,
 *   SUB and MUL wrap, AND / OR / XOR are bitwise, MIN / MAX as named, and EQ, NE, LT, LE, GT and GE give 0 or 1.  An
 *   empty track may have no runs: n_a == n_b == 0 writes *n_out = 0 and out_starts[0] = 0; one of them 0 is
 *   BNPK_E_BADARG.  workspace as for bnpk_row_offsets with n := n_a + n_b.
 * bnpk_interval_intersect: the reference's sorted sweep (intersect / count_overlap, arithmetics/intervals.py:307-335).
 *   start[0 .. n) is sorted inside each segment (segments as for bnpk_interval_merge; same_prev NULL: one segment) and
 *   stop[0 .. n) is the same rows' stops sorted on their own inside each segment.  For every row r + 1 of r's segment
 *   with stop[r] > start[r + 1], in order: out_rows[g] = r + 1, out_stops[g] = stop[r]; *n_out = the number of such
 *   rows.  overlap (int64[1], may be NULL) = the sum of stop[r] - start[r + 1] over them (int64, wrapping).  out_rows
 *   NULL writes only n_out and overlap.  workspace as for bnpk_row_offsets with n := n.
 * BNPK_E_BADARG before any device work for an unknown mode or operator, a size or distance outside [0, 2^59), and a
 * missing pointer the call needs.
 * ------------------------------------------------------------------------------------- */
#define BNPK_PILEUP_COUNT 0
#define BNPK_PILEUP_ANY   1
#define BNPK_RUNS_MAX 0
#define BNPK_RUNS_MIN 1
#define BNPK_RUNS_SUM 2
#define BNPK_RUNS_ANY 3
#define BNPK_OP_ADD 0
#define BNPK_OP_SUB 1
#define BNPK_OP_MUL 2
#define BNPK_OP_AND 3
#define BNPK_OP_OR  4
#define BNPK_OP_XOR 5
#define BNPK_OP_MIN 6
#define BNPK_OP_MAX 7
#define BNPK_OP_EQ  8
#define BNPK_OP_NE  9
#define BNPK_OP_LT  10
#define BNPK_OP_LE  11
#define BNPK_OP_GT  12
#define BNPK_OP_GE  13

int bnpk_interval_events(const int64_t *start, const int64_t *stop, const int32_t *ids, const int64_t *contig_offset,
                         const int64_t *contig_len, size_t n_contigs, int64_t size, size_t n_rows, int64_t *keys,
                         int64_t *g_start, int64_t *g_stop, int64_t *status, void *stream);
int bnpk_pileup_runs(const int64_t *keys, size_t n_keys, int64_t size, int mode, int64_t *run_starts,
                     int64_t *run_values, int64_t *n_runs, void *workspace, size_t workspace_bytes, void *stream);
int bnpk_runs_reduce(const int64_t *run_starts, const int64_t *values, size_t n_runs, const int64_t *q_start,
                     const int64_t *q_stop, size_t n_q, int mode, int64_t *out, int64_t *scratch, void *workspace,
                     size_t workspace_bytes, void *stream);
int bnpk_runs_extract(const int64_t *run_starts, const int64_t *values, size_t n_runs, const int64_t *q_start,
                      size_t n_q, const int64_t *out_offsets, int64_t *out, void *stream);
int bnpk_interval_merge(const int64_t *start, const int64_t *stop, const uint8_t *same_prev, size_t n_rows,
                        int64_t distance, int64_t *out_rows, int64_t *out_stops, int64_t *n_out, int64_t *status,
                        void *workspace, size_t workspace_bytes, void *stream);
int bnpk_rows_equal_prev(const uint8_t *base, size_t base_bytes, const int64_t *starts, const int32_t *lens,
                         size_t n_rows, uint8_t *flag, void *stream);
int bnpk_runs_combine(const int64_t *a_starts, const int64_t *a_values, size_t n_a, const int64_t *b_starts,
                      const int64_t *b_values, size_t n_b, int op, int64_t *out_starts, int64_t *out_values,
                      int64_t *n_out, void *workspace, size_t workspace_bytes, void *stream);
int bnpk_interval_intersect(const int64_t *start, const int64_t *stop, const uint8_t *same_prev, size_t n,
                            int64_t *out_rows, int64_t *out_stops, int64_t *n_out, int64_t *overlap, void *workspace,
                            size_t workspace_bytes, void *stream);

/* K13  a track back into interval rows (GenomicIntervals.from_track, genomic_data/genomic_intervals.py:529-543;
 *   GenomicArray.get_data / _get_intervals_from_data, genomic_data/genomic_track.py:84-91,199-218).
 *   The track is n_runs runs of a global layout (run_starts int64[R + 1], values int64[R], every run non-empty) and
 *   contig_ends int64[C + 1] are the ends of the contigs in it: contig_ends[0] = 0, strictly increasing (a contig of
 *   size 0 has no positions: leave it out), contig_ends[C] = run_starts[R].  A row is one piece of the track inside one
 *   contig, in order: out_contig[g] (int32, index into contig_ends), out_start[g], out_stop[g] (global) and, in
 *   BNPK_RUNS_TO_ALL mode, out_value[g].
 *     BNPK_RUNS_TO_NONZERO  the maximal stretches of non-zero value, cut at contig borders (out_value not written,
 *                           may be NULL): neighbouring non-zero runs are one row whatever their values
 *     BNPK_RUNS_TO_ALL      every run, cut at contig borders (bedGraph)
 *   *n_out = the row count (int64).  Capacity of every output: n_runs + n_contigs rows.  workspace as for
 *   bnpk_row_offsets with n := n_runs.  BNPK_E_BADARG for an unknown mode, n_contigs < 1 with n_runs > 0 and a
 *   missing pointer. */
#define BNPK_RUNS_TO_NONZERO 0
#define BNPK_RUNS_TO_ALL     1
int bnpk_runs_to_intervals(const int64_t *run_starts, const int64_t *values, size_t n_runs, const int64_t *contig_ends,
                           size_t n_contigs, int mode, int32_t *out_contig, int64_t *out_start, int64_t *out_stop,
                           int64_t *out_value, int64_t *n_out, void *workspace, size_t workspace_bytes, void *stream);

/* Bloom filter over k-mer hashes (sequence/bloom_filter.py:15-42): hash function i is v ^ offsets[i]; the filter is
 * one byte per position (the reference's bool mask).  insert: mask[(v ^ offsets[i]) % mask_size] = 1 for every value and
 * function; query: out[j] = AND over the functions. */
int bnpk_bloom_insert(const int64_t *values, size_t n, const int64_t *offsets, int n_hash, uint8_t *mask, size_t mask_size,
                      void *stream);
int bnpk_bloom_query(const int64_t *values, size_t n, const int64_t *offsets, int n_hash, const uint8_t *mask, size_t mask_size,
                     uint8_t *out, void *stream);

/* ---------------------------------------------------------------------------------------
 * Writers: records -> file text (FastQBuffer.from_data / join_fields io/fastq_buffer.py:47-61,
 * OneLineBuffer.join_fields io/one_line_buffer.py:119-134, MultiLineFastaBuffer.from_data
 * io/multiline_buffer.py:67-86).  Entry e with name, sequence and quality lengths Ln, Ls, Lq is
 *   BNPK_FMT_FASTQ          '@' name '\n' seq '\n' '+' '\n' qual '\n'            Ln + Ls + Lq + 6 bytes
 *   BNPK_FMT_FASTA          '>' name '\n' seq '\n'                               Ln + Ls + 3
 *   BNPK_FMT_FASTA_WRAPPED  '>' name '\n', then ceil(Ls / W) lines of W = line_width bases (the last one
 *                           shorter), each ending in '\n'; an empty sequence gives no line
 *                                                                                Ln + 2 + Ls + ceil(Ls / W)
 * `fields` is a HOST array of three bnpk_field: name, sequence, quality (the quality is read by the
 * FASTQ format only).  A field is the ragged view every row kernel takes, rows (base, starts[E],
 * lens[E]); a byte outside [base, base + base_bytes) is written as lut256[0] (never read); lut256 (device, 256 bytes) NULL = copy the bytes, else each byte b is written as
 * lut256[b] (an AlphabetEncoding's codes -> letters; qualities: (v + 33) & 255).
 * Neither entry point traps on bad data.  BNPK_E_BADARG before any device work for an unknown format,
 * line_width < 1 on the wrapped format, a missing name/sequence field (or quality field for FASTQ)
 * when n_entries > 0, and, for bnpk_format_records, out_begin < 0, out_end < out_begin or a NULL out
 * with a non-empty range.
 * ------------------------------------------------------------------------------------- */
#define BNPK_FMT_FASTQ         0
#define BNPK_FMT_FASTA         1
#define BNPK_FMT_FASTA_WRAPPED 2

typedef struct bnpk_field {
    const uint8_t *base;
    size_t base_bytes;
    const int64_t *starts;     /* int64[E] */
    const int32_t *lens;       /* int32[E] (negative = 0) */
    const uint8_t *lut256;     /* NULL or a device 256-byte table */
} bnpk_field;

/* out_offsets int64[E+1]: the exclusive prefix sum of the entry sizes, out_offsets[E] = the text's size (int64: a
 * wrapped chromosome with a long name can exceed int32).  When the sequence field has a LUT, also reads every sequence
 * byte once: the first byte b with lut256[b] == 0 is reported as (entry << 32 | position) in status[BNPK_ST_BAD_BASE]
 * (status pre-initialised; EncodingError(offset), encodings/alphabet_encoding.py:34-46).  Raw text is not read.
 * workspace as for bnpk_row_offsets with n := E. */
int bnpk_format_offsets(int format, int line_width, size_t n_entries, const bnpk_field *fields, int64_t *out_offsets,
                        int64_t *status, void *workspace, size_t workspace_bytes, void *stream);
/* Bytes [out_begin, out_end) of the text whose offsets bnpk_format_offsets made, written to out[0 .. out_end -
 * out_begin).  Any range may be asked for, so a large text can be formatted in slices. */
int bnpk_format_records(int format, int line_width, size_t n_entries, const bnpk_field *fields,
                        const int64_t *out_offsets, int64_t out_begin, int64_t out_end, uint8_t *out, void *stream);

/* K14  delimited text from columns (dump_csv / join_columns, io/dump_csv.py, io/strops.py:186-215): line e is its
 *   columns joined by '\t' and ended by '\n'.  `columns` is a HOST array of n_columns (1..BNPK_MAX_OUT_COLUMNS)
 *   bnpk_out_column, each with E rows, written as its kind says (the reader's column kinds):
 *     BNPK_COL_TEXT    the bytes base[starts[e] .. + lens[e]) (negative length = empty; a byte outside
 *                      [base, base + base_bytes) is written as 0), copied as they are
 *     BNPK_COL_INT     values[e] (int64) in decimal: '-' for a negative value, no leading zero, 0 as "0"
 *     BNPK_COL_STRAND  codes[e] (uint8, StrandEncoding) as '+' (0), '-' (1), '.' (2); another code is written as '.'
 *                      and reported by bnpk_delimited_offsets
 *   bnpk_delimited_offsets: out_offsets int64[E + 1], the exclusive prefix sum of the line sizes (out_offsets[E] = the
 *   text's size); the first bad strand code is atomicMin-ed into status[BNPK_ST_BAD_BASE] as (line << 8 | column << 3
 *   | BNPK_BAD_STRAND) (status pre-initialised).  workspace as for bnpk_row_offsets with n := E.
 *   bnpk_delimited_format: bytes [out_begin, out_end) of that text written to out[0 .. out_end - out_begin), as
 *   bnpk_format_records.  BNPK_E_BADARG before any device work for a bad column count or kind, a missing pointer,
 *   out_begin < 0 or out_end < out_begin. */
#define BNPK_MAX_OUT_COLUMNS 8

typedef struct bnpk_out_column {
    int kind;
    const void *data;          /* TEXT: base bytes; INT: int64[E]; STRAND: uint8[E] */
    size_t base_bytes;         /* TEXT */
    const int64_t *starts;     /* TEXT: int64[E] */
    const int32_t *lens;       /* TEXT: int32[E] */
} bnpk_out_column;

int bnpk_delimited_offsets(const bnpk_out_column *columns, int n_columns, size_t n_lines, int64_t *out_offsets,
                           int64_t *status, void *workspace, size_t workspace_bytes, void *stream);
int bnpk_delimited_format(const bnpk_out_column *columns, int n_columns, size_t n_lines, const int64_t *out_offsets,
                          int64_t out_begin, int64_t out_end, uint8_t *out, void *stream);

/* ---------------------------------------------------------------------------------------
 * K15  BAM records (BamBuffer._find_starts / BamBufferExtractor, io/bam.py:18-331; split_cigar /
 * count_reference_length, alignments/cigar.py:8-24).  `chunk` holds inflated BAM bytes that start at a record.
 *
 *   bnpk_bam_split: the byte offset of every complete record of the chunk, in order, into starts int64[R]
 *     (max_starts >= n / 36: a complete record is at least 36 bytes).  A speculative segmented walk: the chunk is cut
 *     into segments of segment_bytes; a warp per segment finds the first offset whose record header (and the next
 *     few records of its chain) passes the header check and walks from there to the segment's end; one warp then
 *     confirms the segments in order from offset 0, walking again every segment whose speculative start is not the
 *     confirmed exit of the segment before.  The result is exact whatever the speculation found.  The header check:
 *     block_size >= 32, -1 <= refID, next_refID < n_ref, l_read_name >= 1 and the name ends in NUL, and
 *     32 + l_read_name + 4 n_cigar_op + (l_seq + 1) / 2 + l_seq <= block_size with l_seq >= 0.
 *     status (pre-initialised): [BNPK_ST_N_RECORDS] = R, [BNPK_ST_N_COMPLETE_BYTES] = the bytes of those records (the
 *     rest begins the next chunk's first record), [BNPK_ST_BAD_BASE] = (R << 8 | BNPK_BAM_BAD_*) when the walk
 *     stopped at a record that fails the check, [BNPK_ST_N_VALUES] = the segments walked again.  workspace int64[7 *
 *     ceil(n / segment_bytes)]; three kernels, no synchronisation.
 *   bnpk_bam_fields: one thread per record r < min(max_records, status[BNPK_ST_N_RECORDS]) writes
 *     fields[f * max_records + r] for the BNPK_BAM_F_* below, and atomicMin-s (r << 8 | BNPK_BAM_BAD_CIGAR_OP) into
 *     status[BNPK_ST_BAD_BASE] for a cigar op code above 8.  The records are those bnpk_bam_split found.
 *   bnpk_bam_sequence: the l_seq 4-bit codes of every row, high nibble first, one byte each, at out[offsets[r] ..
 *     offsets[r + 1]) (offsets = bnpk_row_offsets of l_seq); 16 output bytes per thread.
 *   bnpk_bam_cigar: the n_cigar_op cigar words of every row as op = word & 15 (uint8) and length = word >> 4 (int64)
 *     at offsets[r] .. offsets[r + 1]; 4 ops per thread.
 * ------------------------------------------------------------------------------------- */
#define BNPK_BAM_BAD_BLOCK_SIZE 1  /* block_size < 32                                             */
#define BNPK_BAM_BAD_REF_ID     2  /* refID or next_refID outside -1 .. n_ref - 1                 */
#define BNPK_BAM_BAD_NAME       3  /* l_read_name 0, or the name does not end in NUL              */
#define BNPK_BAM_BAD_SIZES      4  /* l_seq < 0, or the fields do not fit block_size              */
#define BNPK_BAM_BAD_CIGAR_OP   5  /* a cigar op code above 8 (MIDNSHP=X)                         */
#define BNPK_BAM_TRUNCATED      6  /* the file ends inside a record (reported by the reader)      */
#define BNPK_BAM_F_REF_ID     0
#define BNPK_BAM_F_POS        1
#define BNPK_BAM_F_MAPQ       2
#define BNPK_BAM_F_FLAG       3
#define BNPK_BAM_F_NAME_START 4    /* the name without its NUL: l_read_name - 1 bytes             */
#define BNPK_BAM_F_NAME_LEN   5
#define BNPK_BAM_F_CIGAR_START 6
#define BNPK_BAM_F_N_CIGAR    7
#define BNPK_BAM_F_SEQ_START  8
#define BNPK_BAM_F_L_SEQ      9
#define BNPK_BAM_F_QUAL_START 10   /* l_seq bytes                                                 */
#define BNPK_BAM_F_REF_LEN    11   /* the summed lengths of the M, D, N, = and X ops              */
#define BNPK_BAM_FIELDS       12

int bnpk_bam_split(const uint8_t *chunk, size_t n, int n_ref, size_t segment_bytes, int64_t *starts, size_t max_starts,
                   int64_t *status, int64_t *workspace, size_t workspace_words, void *stream);
int bnpk_bam_fields(const uint8_t *chunk, size_t n, const int64_t *starts, size_t max_records, int64_t *fields,
                    int64_t *status, void *stream);
int bnpk_bam_sequence(const uint8_t *chunk, size_t n, const int64_t *seq_start, const int64_t *offsets, size_t n_rows,
                      uint8_t *out, void *stream);
int bnpk_bam_cigar(const uint8_t *chunk, size_t n, const int64_t *cigar_start, const int64_t *offsets, size_t n_rows,
                   uint8_t *op, int64_t *length, void *stream);

/* ---------------------------------------------------------------------------------------
 * Host-buffer entry point (end-to-end): the call a reader loop makes with a chunk that is
 * still in host memory.  Copies `chunk_host` (pinned or pageable) to the device in slices on
 * a private copy stream, overlapping each slice's H2D with the fused count of the previous
 * one, accumulates into the DEVICE histogram `hist`, and copies the status block back to
 * `status_host` (int64[BNPK_ST_WORDS]).  Synchronises before returning.
 * Replaces CupyFileReader._get_buffer's cp.asanyarray(chunk) (cupy_compatible/parser.py:11-17)
 * plus the K6 chain above.  `ctx` comes from bnpk_pipeline_create (owns the device staging
 * buffer, workspace, streams, events); capacity = largest chunk it will be given.
 * ------------------------------------------------------------------------------------- */
typedef struct bnpk_pipeline bnpk_pipeline;
int  bnpk_pipeline_create(bnpk_pipeline **ctx, size_t capacity_bytes, size_t slice_bytes);
void bnpk_pipeline_destroy(bnpk_pipeline *ctx);
int  bnpk_pipeline_kmer_count_host(bnpk_pipeline *ctx, const uint8_t *chunk_host, size_t n,
                                   int lines_per_entry, uint8_t header_char, int check_plus, int trim_cr,
                                   int enc_mode, const uint8_t *lut256_host, int k, int window_size,
                                   int64_t n_bins, int hist_mode, int64_t *hist, int64_t *status_host);
/* The same, ordered after the work already queued on `stream` (whatever produced or zeroed `hist`); the entry point
 * above orders itself after the legacy default stream. */
int  bnpk_pipeline_kmer_count_host_on(bnpk_pipeline *ctx, const uint8_t *chunk_host, size_t n,
                                      int lines_per_entry, uint8_t header_char, int check_plus, int trim_cr,
                                      int enc_mode, const uint8_t *lut256_host, int k, int window_size,
                                      int64_t n_bins, int hist_mode, int64_t *hist, int64_t *status_host, void *stream);

/* ---------------------------------------------------------------------------------------
 * Synthetic workload generator (SURVEY 8d record: "@r%010d\n" + 150 bases + "\n+\n" +
 * 150*'I' + "\n" = 317 B), bit-identical to oracle/bnp_oracle.py:synthetic_fastq.
 * Test/bench utility; out must hold n_records*317 bytes.
 * ------------------------------------------------------------------------------------- */
int bnpk_synth_fastq(uint8_t *out, uint64_t first_record, uint64_t n_records, uint64_t seed, void *stream);

/* Measurement hooks: when enabled, every launch of the dominant (tile) kernel is bracketed by
 * CUDA events on the launching stream; bnpk_profile_read waits for them, returns the summed
 * duration and the launch count, and clears the list. */
int bnpk_profile_enable(int on);
int bnpk_profile_read(double *total_ms, uint64_t *n_launches);

/* how many kernels this library has launched in this process (bench's gpu_launches) */
uint64_t bnpk_launch_count(void);

#ifdef __cplusplus
}
#endif
#endif /* BNPK_H */
