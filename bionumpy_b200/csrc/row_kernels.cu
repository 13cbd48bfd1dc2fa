// row_kernels.cu -- kernels driven by a row-offset vector (starts[R], lens[R]) over a byte buffer:
// the general EncodedRaggedArray form (io/file_buffers.py:335-338).  One warp per read row; rows
// longer than one staging segment are walked in overlapping segments by the same warp.
//   K2 rows_encode      change_encoding            encoded_array.py:655-695
//   K3 rows_kmer_hash   get_kmers/_get_dna_kmers   sequence/kmers.py:36-126
//   K4 rows_minimizers  get_minimizers             sequence/minimizers.py:20-54
//   K3/K4+K5 rows_kmer_count   count_kmers         sequence/kmers.py:129-145
//   K3 + table rows_kmer_table_insert  exact distinct-k-mer counts (extension, like `jellyfish count`)
//   K7 rows_pwm_scores / rows_pwm_max  get_motif_scores, PWM.calculate_scores  sequence/position_weight_matrix.py:83-100,166-196
//   K8 rows_match / rows_match_count   match_string, StringMatcher, RegexMatcher  sequence/string_matcher.py
// plus the clean-up passes of the fused chunk count (long rows, trailing incomplete entry).
#include <climits>
#include "bnpk_host.h"

namespace bnpk {

constexpr int kRowThreads = 256;
constexpr int kRowWarps = kRowThreads / 32;
constexpr int kSegUnits = 128;               // 2 KiB staged per warp and segment
constexpr int kSegBytes = kSegUnits * 16;
constexpr int kWarpWords = 2 * kSegUnits + 4;

enum { RM_ENCODE = 0, RM_HASH = 1, RM_MINIMIZER = 2, RM_COUNT = 3, RM_COUNT_MIN = 4, RM_TABLE = 5, RM_PWM = 6,
       RM_PWM_MAX = 7, RM_MATCH = 8, RM_MATCH_COUNT = 9 };
constexpr int kPwmMaxLen = kSegBytes / 2;     // motif columns: the segment overlap limit of check_common
constexpr int kPwmMaxCells = 8192;            // alphabet_size * motif_len doubles: 64 KiB of shared memory
constexpr int kPwmInFlight = 4;               // positions per lane summed side by side (each one a chain of DADDs)
constexpr int kMatchMaxLen = kSegBytes / 2;   // columns of one sub-pattern: the segment overlap, as check_common
constexpr int kMatchMaxSubs = 64;             // sub-patterns of one expanded pattern
constexpr int kMatchMaxWords = 8192;          // symbol-set words of all columns: 32 KiB of shared memory

// A pattern expanded into sub-patterns (one per combination of gap lengths), the match of a position being the OR of
// theirs.  Column c of the concatenated sub-patterns is the symbol set sets[c * words_per_col ...]: bit s of the
// words is set when code s (a byte, for raw bytes) matches there.
struct MatchArgs {
    const uint32_t *sets;
    int n_sub, span, words_per_col, n_words, same;
    int len[kMatchMaxSubs];
};
// The match modes' shared memory behind the LUT: [kMatchMaxSubs] lengths, [kMatchMaxSubs] first columns, then the sets.
constexpr int kMatchSmemHead = 2 * kMatchMaxSubs * 4;

struct RowArgs {
    const uint8_t *base;
    size_t base_bytes;
    const int64_t *starts;
    const int32_t *lens;
    size_t n_rows;
    const uint8_t *lut;
    int k, window;
    const int64_t *offsets;
    void *out;
    uint64_t n_bins;
    unsigned long long *hist;
    int64_t *status;
    // deferred (long-row) mode
    const uint64_t *deferred_count;
    const uint64_t *deferred;
    size_t deferred_cap;
    int lpe;
    uint64_t canon_xor;          // != 0: canonical k-mers (hash / count / table modes without a minimizer window)
    KmerTable table;             // table mode
    // motif modes: matrix[j * 4 + c] (motif_len = window), and whether the last window - 1 positions of a row are
    // scored with the columns that fit
    const double *pwm;
    int tail;
};

// NaN-propagating maximum (np.max): once a NaN is in, it stays
__device__ __forceinline__ double nan_max(double m, double v) { return (v > m || v != v) ? v : m; }

// Motif scores of the positions of one staged segment that start in [0, npos): s = +0.0, then s += table[j][code]
// for j = 0, 1, ... in order (PWM.calculate_scores, sequence/position_weight_matrix.py:96-99), each position with the
// columns that fit before seg_len.  Codes come 16 at a time from the packed stream.  Writes out[p] (SCORES) or folds
// the scores into `best`.  Returns the positions this lane scored.  Warp-wide.
template <bool SCORES>
__device__ __forceinline__ uint32_t pwm_segment(const uint32_t *w_codes, const double *s_pwm, int off, int seg_len,
                                                int npos, int m, double *out, double &best, int lane) {
    uint32_t produced = 0;
    for (int p0 = lane; p0 < npos; p0 += 32 * kPwmInFlight) {
        double s[kPwmInFlight];
        int nc[kPwmInFlight];
#pragma unroll
        for (int q = 0; q < kPwmInFlight; ++q) {
            const int p = p0 + 32 * q;
            nc[q] = p < npos ? min(m, seg_len - p) : 0;
            s[q] = 0.0;
        }
        for (int jb = 0; jb < nc[0]; jb += 16) {
            uint32_t w[kPwmInFlight];
#pragma unroll
            for (int q = 0; q < kPwmInFlight; ++q)
                w[q] = jb < nc[q] ? stream_lo32(w_codes, (uint32_t)(off + p0 + 32 * q + jb)) : 0u;
            const int je = min(16, nc[0] - jb);
            for (int jj = 0; jj < je; ++jj) {
                const double *col = s_pwm + 4 * (jb + jj);
#pragma unroll
                for (int q = 0; q < kPwmInFlight; ++q)
                    if (jb + jj < nc[q]) s[q] += col[(w[q] >> (2 * jj)) & 3u];
            }
        }
#pragma unroll
        for (int q = 0; q < kPwmInFlight; ++q) {
            const int p = p0 + 32 * q;
            if (p < npos) {
                if constexpr (SCORES) out[p] = s[q];
                else best = nan_max(best, s[q]);
                ++produced;
            }
        }
    }
    return produced;
}

// Whether each of 16 2-bit codes (code i at bits 2i, 2i+1 of y) is in the 4-letter set s (bit c = code c), as bit 2i of
// the result: the set's truth table over the word's two bit planes.  Odd bits are don't-care.
__device__ __forceinline__ uint32_t codes_in_set(uint32_t y, uint32_t s) {
    const uint32_t lo = y, hi = y >> 1;
    const uint32_t s0 = 0u - (s & 1u), s1 = 0u - ((s >> 1) & 1u), s2 = 0u - ((s >> 2) & 1u), s3 = 0u - (s >> 3);
    return (~hi & ((~lo & s0) | (lo & s1))) | (hi & ((~lo & s2) | (lo & s3)));
}

// Matches at the positions of one staged segment that start in [0, npos), 16 starts per lane at a time: bit 2i of a
// sub-pattern's word is start p0 + i, ANDed over the sub-pattern's columns (codes p0 + j .. p0 + j + 15 come from the
// packed stream in one funnel shift) and ORed over the sub-patterns.  A start only counts for a sub-pattern that fits
// before seg_len; '.' columns (all four codes) are skipped, and a sub-pattern whose 16 starts have all failed stops.
// Writes out[p] = 0/1 (OUT) and adds the matches to `hits`.  Returns the positions this lane tested.  Warp-wide.
template <bool OUT>
__device__ __forceinline__ uint32_t match_segment(const uint32_t *w_codes, const int *s_match, int n_sub, int off,
                                                  int seg_len, int npos, uint8_t *out, uint64_t &hits, int lane) {
    const uint32_t *s_sets = reinterpret_cast<const uint32_t *>(s_match + 2 * kMatchMaxSubs);
    uint32_t produced = 0;
    for (int p0 = 16 * lane; p0 < npos; p0 += 16 * 32) {
        const int nv = min(16, npos - p0);
        uint32_t any = 0;
        for (int k = 0; k < n_sub; ++k) {
            const int m = s_match[k];
            const int fit = min(nv, seg_len - m + 1 - p0);           // starts of the block where sub-pattern k fits
            if (fit <= 0) continue;
            uint32_t acc = 0x55555555u >> (32 - 2 * fit);
            const uint32_t *set = s_sets + s_match[kMatchMaxSubs + k];
            for (int j = 0; j < m && acc; ++j) {
                const uint32_t s = set[j];
                if (s == 0xFu) continue;
                acc &= codes_in_set(stream_lo32(w_codes, (uint32_t)(off + p0 + j)), s);
            }
            any |= acc;
        }
        if constexpr (OUT)
            for (int i = 0; i < nv; ++i) out[p0 + i] = (uint8_t)((any >> (2 * i)) & 1u);
        hits += (uint64_t)__popc(any);
        produced += (uint32_t)nv;
    }
    return produced;
}

template <int RM, int ENC, bool SMEM_HIST>
__device__ void warp_row(const RowArgs &a, uint32_t *w_codes, uint32_t *w_bad, const uint8_t *s_lut,
                         const HistTarget &ht, int64_t start, int64_t L, int64_t r, int64_t out_off, int lane,
                         uint64_t &acc_values, uint64_t *acc_claims = nullptr, const double *s_pwm = nullptr,
                         const MatchArgs *ma = nullptr, const int *s_match = nullptr) {
    constexpr bool MINZ = (RM == RM_MINIMIZER || RM == RM_COUNT_MIN);
    constexpr bool PWM = (RM == RM_PWM || RM == RM_PWM_MAX);
    constexpr bool MATCH = (RM == RM_MATCH || RM == RM_MATCH_COUNT);
    constexpr bool LUT_ENCODE = RM == RM_ENCODE && ENC == BNPK_ENC_LUT;   // writes the table values, finds its own bad bytes
    const int span = (MINZ || PWM || MATCH) ? a.window : (RM == RM_ENCODE ? 1 : a.k);
    double best = -INFINITY;                                              // RM_PWM_MAX: this lane's maximum
    uint64_t hits = 0;                                                    // RM_MATCH_COUNT: this lane's matches
    const uint64_t kmask = (1ull << (2 * a.k)) - 1;
    int64_t seg_start = 0;
    bool reported = false;
    while (seg_start < L) {
        const int64_t g0 = start + seg_start;
        const int off = (int)((reinterpret_cast<uintptr_t>(a.base) + g0) & 15);
        const int64_t ua = g0 - off;
        const int seg_len = (int)min(L - seg_start, (int64_t)(kSegBytes - off));
        const int n_units = (off + seg_len + 15) >> 4;
        if constexpr (!LUT_ENCODE) {
            for (int u = lane; u < n_units; u += 32) {
                const uint4 q = load_unit_guarded(a.base, a.base_bytes, ua + 16 * (int64_t)u);
                uint32_t bad;
                w_codes[u] = encode_unit<ENC, false>(q, 0xFFFFu, s_lut, bad);
                w_bad[u] = bad;
            }
            if (lane < 4) w_codes[n_units + lane] = 0;
        }
        __syncwarp();
        if (!reported && !LUT_ENCODE) {
            const int bad = find_invalid(w_bad, off, off + seg_len, lane);
            if (bad >= 0) {
                reported = true;
                if (lane == 0)
                    report_fault(a.status, fault_row_pos(r, seg_start + bad - off));
            }
        }
        if constexpr (RM == RM_ENCODE) {
            uint8_t *out = reinterpret_cast<uint8_t *>(a.out) + out_off + seg_start;
            if constexpr (ENC == BNPK_ENC_LUT) {
                // any alphabet size: the full LUT value is the code, 255 = invalid
                // (AlphabetEncoding._encode, encodings/alphabet_encoding.py:34-46)
                int first_bad = INT_MAX;
                for (int p = lane; p < seg_len; p += 32) {
                    const uint8_t code = s_lut[a.base[g0 + p]];
                    out[p] = code;
                    if (code == 255 && p < first_bad) first_bad = p;
                }
#pragma unroll
                for (int o = 16; o; o >>= 1) first_bad = min(first_bad, __shfl_xor_sync(0xffffffffu, first_bad, o));
                if (first_bad != INT_MAX && !reported) {
                    reported = true;
                    if (lane == 0)
                        report_fault(a.status, fault_row_pos(r, seg_start + first_bad));
                }
            } else {
                for (int p = lane; p < seg_len; p += 32) {
                    const int b = off + p;
                    out[p] = (uint8_t)((w_codes[b >> 4] >> (2 * (b & 15))) & 3u);
                }
            }
        } else if constexpr (RM == RM_HASH) {
            int64_t *out = reinterpret_cast<int64_t *>(a.out) + out_off + seg_start;
            const int npos = seg_len - span + 1;
            for (int p = lane; p < npos; p += 32) {
                uint64_t h = stream_64(w_codes, (uint32_t)(off + p)) & kmask;
                if (a.canon_xor) h = canonical_hash(h, a.k, a.canon_xor);
                out[p] = (int64_t)h;
            }
            if (npos > 0) acc_values += (uint64_t)((npos - lane + 31) / 32);
        } else if constexpr (RM == RM_TABLE) {
            // the k-mers of RM_HASH, inserted into the table instead of written out
            const int npos = seg_len - span + 1;
            uint32_t claimed = 0;
            for (int p = lane; p < npos; p += 32) {
                uint64_t h = stream_64(w_codes, (uint32_t)(off + p)) & kmask;
                if (a.canon_xor) h = canonical_hash(h, a.k, a.canon_xor);
                claimed += table_insert(a.table, h, 1ull, a.status);
            }
            if (npos > 0) acc_values += (uint64_t)((npos - lane + 31) / 32);
            *acc_claims += claimed;
        } else if constexpr (RM == RM_MINIMIZER) {
            int64_t *out = reinterpret_cast<int64_t *>(a.out) + out_off + seg_start;
            const int w = a.window - a.k + 1;
            const int nout = seg_len - a.window + 1;
            const int nh = seg_len - a.k + 1;
            if (w <= 32) {
                const int step = 32 - (w - 1);
                for (int base = 0; base < nout; base += step) {
                    const int p = base + lane;
                    uint64_t h = ~0ull;
                    if (p < nh) h = stream_64(w_codes, (uint32_t)(off + p)) & kmask;
                    const uint64_t m = warp_sliding_min(h, w);
                    if (lane < step && p < nout) { out[p] = (int64_t)m; ++acc_values; }
                }
            } else {
                for (int j = lane; j < nout; j += 32) {
                    uint64_t m = ~0ull;
                    for (int i = 0; i < w; ++i) {
                        const uint64_t h = stream_64(w_codes, (uint32_t)(off + j + i)) & kmask;
                        m = h < m ? h : m;
                    }
                    out[j] = (int64_t)m;
                    ++acc_values;
                }
            }
        } else if constexpr (PWM) {
            // with `tail`, the row's last segment also scores its last span - 1 positions with the columns that fit
            const int npos = (a.tail && seg_start + seg_len >= L) ? seg_len : seg_len - span + 1;
            acc_values += pwm_segment<RM == RM_PWM>(w_codes, s_pwm, off, seg_len, npos, span,
                                                    reinterpret_cast<double *>(a.out) + out_off + seg_start, best, lane);
        } else if constexpr (MATCH) {
            // "same": the row's last segment also tests its last span - 1 positions, with the sub-patterns that fit
            const int npos = (ma->same && seg_start + seg_len >= L) ? seg_len : seg_len - span + 1;
            acc_values += match_segment<RM == RM_MATCH>(w_codes, s_match, ma->n_sub, off, seg_len, npos,
                                                        reinterpret_cast<uint8_t *>(a.out) + out_off + seg_start, hits,
                                                        lane);
        } else {
            if (seg_len >= span)
                acc_values += row_count<SMEM_HIST, MINZ>(w_codes, off, seg_len, a.k, a.window, ht, lane);
        }
        __syncwarp();
        if (seg_start + seg_len >= L) break;
        seg_start += seg_len - (span - 1);
    }
    if constexpr (RM == RM_PWM_MAX) {
#pragma unroll
        for (int o = 16; o; o >>= 1) best = nan_max(best, __shfl_xor_sync(0xffffffffu, best, o));
        if (lane == 0) reinterpret_cast<double *>(a.out)[r] = best;
    }
    if constexpr (RM == RM_MATCH_COUNT) {
        hits = warp_sum_u64(hits);
        if (lane == 0) reinterpret_cast<int64_t *>(a.out)[r] = (int64_t)hits;
    }
}

// The body of the row kernels: one warp per row, the block's rows strided over the grid.
template <int RM, int ENC, bool SMEM_HIST, bool DEFERRED>
__device__ __forceinline__ void rows_body(const RowArgs &a, const MatchArgs *ma = nullptr) {
    extern __shared__ __align__(16) uint32_t smem[];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    uint32_t *w_codes = smem + warp * kWarpWords;
    uint32_t *w_bad = w_codes + kSegUnits + 4;
    uint8_t *s_lut = reinterpret_cast<uint8_t *>(smem + kRowWarps * kWarpWords);
    uint32_t *s_hist = reinterpret_cast<uint32_t *>(s_lut + 256);
    double *s_pwm = reinterpret_cast<double *>(s_lut + 256);              // motif modes: the [window][4] table
    if (ENC == BNPK_ENC_LUT && tid < 256) s_lut[tid] = a.lut[tid];
    constexpr bool PWM = (RM == RM_PWM || RM == RM_PWM_MAX);
    if constexpr (PWM)
        for (int i = tid; i < 4 * a.window; i += kRowThreads) s_pwm[i] = a.pwm[i];
    constexpr bool MATCH = (RM == RM_MATCH || RM == RM_MATCH_COUNT);
    int *s_match = reinterpret_cast<int *>(s_lut + 256);                   // match modes: kMatchSmemHead, then the sets
    if constexpr (MATCH) {
        if (tid == 0) {
            int col = 0;
#pragma unroll
            for (int k = 0; k < kMatchMaxSubs; ++k)
                if (k < ma->n_sub) { s_match[k] = ma->len[k]; s_match[kMatchMaxSubs + k] = col; col += ma->len[k]; }
        }
        uint32_t *s_sets = reinterpret_cast<uint32_t *>(s_match + 2 * kMatchMaxSubs);
        for (int i = tid; i < ma->n_words; i += kRowThreads) s_sets[i] = ma->sets[i];
    }
    constexpr bool COUNTING = (RM == RM_COUNT || RM == RM_COUNT_MIN);
    if (COUNTING && SMEM_HIST)
        for (uint32_t b = tid; b < a.n_bins; b += kRowThreads) s_hist[b] = 0;
    HistTarget ht;
    ht.global = a.hist;
    ht.smem = s_hist;
    ht.n_bins = a.n_bins;
    ht.mask = (a.n_bins & (a.n_bins - 1)) == 0 ? a.n_bins - 1 : 0;
    ht.delta = 1ull;
    ht.canon_xor = a.canon_xor;
    __syncthreads();

    uint64_t acc_values = 0, acc_bases = 0, acc_long = 0, acc_claims = 0;
    size_t n_rows = a.n_rows;
    int64_t n_records = 0;
    bool cr = false;
    if (DEFERRED) {
        n_rows = (size_t)min((unsigned long long)*a.deferred_count, (unsigned long long)a.deferred_cap);
        n_records = a.status[BNPK_ST_N_RECORDS];
        cr = a.status[BNPK_ST_CR] != 0;
    }
    for (size_t row = (size_t)blockIdx.x * kRowWarps + warp; row < n_rows; row += (size_t)gridDim.x * kRowWarps) {
        int64_t start, L, r, out_off = 0;
        if (DEFERRED) {
            start = (int64_t)a.deferred[2 * row];
            r = (int64_t)a.deferred[2 * row + 1];
            if (r >= n_records) continue;                     // belongs to a trailing incomplete entry
            L = warp_line_len(a.base, a.base_bytes, start, lane);
            if (L < 0) continue;
            if (cr && L > 0 && a.base[start + L - 1] == '\r') L -= 1;
            if (lane == 0) ++acc_long;
        } else {
            start = a.starts[row];
            L = a.lens[row];
            r = (int64_t)row;
            if (a.offsets) out_off = a.offsets[row];
        }
        if (L <= 0) {
            if constexpr (RM == RM_PWM_MAX)
                if (lane == 0) reinterpret_cast<double *>(a.out)[r] = -INFINITY;   // no window
            if constexpr (RM == RM_MATCH_COUNT)
                if (lane == 0) reinterpret_cast<int64_t *>(a.out)[r] = 0;
            continue;
        }
        if (lane == 0) acc_bases += (uint64_t)L;
        warp_row<RM, ENC, SMEM_HIST>(a, w_codes, w_bad, s_lut, ht, start, L, r, out_off, lane, acc_values, &acc_claims,
                                     s_pwm, ma, s_match);
    }
    if (COUNTING && SMEM_HIST) {
        __syncthreads();
        for (uint32_t b = tid; b < a.n_bins; b += kRowThreads) {
            const uint32_t c = s_hist[b];
            if (c) atomicAdd(a.hist + b, (unsigned long long)c);
        }
    }
    acc_values = warp_sum_u64(acc_values);
    acc_bases = warp_sum_u64(acc_bases);
    acc_long = warp_sum_u64(acc_long);
    if (lane == 0) {
        if (acc_values) atomicAdd((unsigned long long *)&a.status[BNPK_ST_N_VALUES], acc_values);
        if (acc_bases) atomicAdd((unsigned long long *)&a.status[BNPK_ST_N_BASES], acc_bases);
        if (acc_long) atomicAdd((unsigned long long *)&a.status[BNPK_ST_N_LONG_ROWS], acc_long);
    }
    if constexpr (RM == RM_TABLE) {
        acc_claims = warp_sum_u64(acc_claims);
        if (lane == 0 && acc_claims) atomicAdd(a.table.n_used, (unsigned long long)acc_claims);
    }
}

// Table mode and the long-row minimizer count ask for 4 CTAs per SM (<= 64 registers): without a minimum, ptxas keeps
// the row loop's 64-bit accumulators on the stack (table mode: the code-byte build; long rows: every build).  0 = no
// minimum, the other modes' code is unchanged by it.
template <int RM, int ENC, bool SMEM_HIST, bool DEFERRED>
__global__ void __launch_bounds__(kRowThreads, (RM == RM_TABLE || (RM == RM_COUNT_MIN && DEFERRED)) ? 4 : 0)
rows_kernel(const RowArgs a) {
    rows_body<RM, ENC, SMEM_HIST, DEFERRED>(a);
}

// The motif modes (RM_PWM, RM_PWM_MAX), with 4 CTAs per SM for the same reason (the LUT build of the scores).
template <int RM, int ENC>
__global__ void __launch_bounds__(kRowThreads, 4) rows_pwm_kernel(const RowArgs a) {
    rows_body<RM, ENC, false, false>(a);
}

// The match modes (RM_MATCH, RM_MATCH_COUNT) of four-letter alphabets.  2 CTAs per SM (<= 128 registers): at 4, ptxas
// keeps a 64-bit accumulator of the count on the stack.
template <int RM, int ENC>
__global__ void __launch_bounds__(kRowThreads, 2) rows_match_kernel(const RowArgs a, const __grid_constant__ MatchArgs m) {
    rows_body<RM, ENC, false, false>(a, &m);
}

// Growth: one thread per slot of the old table re-inserts its (key, count) into the new one with the same slot function.
__global__ void __launch_bounds__(256) table_rehash_kernel(const int64_t *keys, const int64_t *counts, size_t capacity,
                                                           const KmerTable t, int64_t *status) {
    uint64_t claimed = 0;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < capacity; i += (size_t)gridDim.x * blockDim.x) {
        const unsigned long long key = (unsigned long long)keys[i];
        if (key != kTableEmpty) claimed += table_insert(t, key, (unsigned long long)counts[i], status);
    }
    claimed = warp_sum_u64(claimed);
    if ((threadIdx.x & 31) == 0 && claimed) atomicAdd(t.n_used, (unsigned long long)claimed);
}

// Un-count the sequence line of a trailing incomplete entry: the fused pass counts every
// terminated sequence line it meets; the reference only keeps entries with all their lines
// (io/one_line_buffer.py:67).  One warp.
template <int ENC, bool MINZ>
__global__ void uncount_kernel(const RowArgs a) {
    extern __shared__ __align__(16) uint32_t smem[];
    const int lane = threadIdx.x & 31;
    const int64_t n_lines = a.status[BNPK_ST_N_LINES];
    const int64_t n_records = n_lines / a.lpe;
    if (n_lines % a.lpe < 2) return;                          // its sequence line was never terminated
    if (a.status[BNPK_ST_LAST_ROW_INDEX] - 1 != n_records) return;  // that line was not counted in-tile
    const int64_t start = a.status[BNPK_ST_LAST_ROW_START] - 1;
    int64_t L = warp_line_len(a.base, a.base_bytes, start, lane);
    if (L < 0) return;
    if (a.status[BNPK_ST_CR] != 0 && L > 0 && a.base[start + L - 1] == '\r') L -= 1;
    uint32_t *w_codes = smem;
    uint32_t *w_bad = w_codes + kSegUnits + 4;
    uint8_t *s_lut = reinterpret_cast<uint8_t *>(smem + kWarpWords);
    if (ENC == BNPK_ENC_LUT)
        for (int i = lane; i < 256; i += 32) s_lut[i] = a.lut[i];
    __syncwarp();
    HistTarget ht;
    ht.global = a.hist;
    ht.smem = nullptr;
    ht.n_bins = a.n_bins;
    ht.mask = (a.n_bins & (a.n_bins - 1)) == 0 ? a.n_bins - 1 : 0;
    ht.delta = ~0ull;                                          // -1
    ht.canon_xor = 0;
    uint64_t produced = 0;
    // the BAD_BASE slot must not be touched by this row: point validation at a scratch word
    RowArgs b = a;
    __shared__ int64_t scratch_status[BNPK_ST_WORDS];
    if (lane < BNPK_ST_WORDS) scratch_status[lane] = INT64_MAX;
    __syncwarp();
    b.status = scratch_status;
    warp_row<MINZ ? RM_COUNT_MIN : RM_COUNT, ENC, false>(b, w_codes, w_bad, s_lut, ht, start, L, n_records, 0, lane, produced);
    produced = warp_sum_u64(produced);
    if (lane == 0) {
        atomicAdd((unsigned long long *)&a.status[BNPK_ST_N_VALUES], 0ull - produced);
        atomicAdd((unsigned long long *)&a.status[BNPK_ST_N_BASES], 0ull - (unsigned long long)L);
    }
}


// ---------------------------------------------------------------------------------------------
// Generic alphabets (size != 4): h = sum_j code[i+j] * A^j in int64 arithmetic, the reference's
// KmerEncoder dot product (sequence/kmers.py:17-27, sequence/rollable.py:49-66).  One warp per row,
// one lane per window; codes come from a 256-byte LUT (or are the bytes themselves).
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) rows_generic_hash_kernel(const uint8_t *base, size_t base_bytes, const int64_t *starts,
                                                                const int32_t *lens, size_t n_rows, const uint8_t *lut,
                                                                int alphabet_size, int k, const int64_t *offsets,
                                                                int64_t *out, int64_t *status) {
    __shared__ uint8_t s_lut[256];
    __shared__ unsigned long long s_pow[64];
    const int tid = threadIdx.x, lane = tid & 31;
    if (tid < 256) s_lut[tid] = lut ? lut[tid] : (uint8_t)tid;
    if (tid == 0) {
        unsigned long long p = 1;
        for (int j = 0; j < 64; ++j) { s_pow[j] = p; p *= (unsigned long long)alphabet_size; }
    }
    __syncthreads();
    const size_t warp_global = ((size_t)blockIdx.x * blockDim.x + tid) >> 5;
    const size_t n_warps = ((size_t)gridDim.x * blockDim.x) >> 5;
    for (size_t r = warp_global; r < n_rows; r += n_warps) {
        const int64_t start = starts[r], L = lens[r], o = offsets[r];
        for (int64_t i = lane; i < L; i += 32) {                    // validity of every symbol of the row
            const uint8_t c = s_lut[base[start + i]];
            if (c >= alphabet_size) report_fault(status, fault_row_pos(r, i));
        }
        for (int64_t i = lane; i + k <= L; i += 32) {
            unsigned long long h = 0;
            for (int j = 0; j < k; ++j) h += (unsigned long long)s_lut[base[start + i + j]] * s_pow[j];
            out[o + i] = (int64_t)h;
        }
    }
}

// Motif scores for alphabets that are not four letters ("ACE", "ACGTN", amino acids): the same sums, tail and maximum as
// rows_kernel's motif modes, with codes from a 256-byte LUT in shared memory (255 = invalid; byte codes: c < A maps to
// itself) and the [m][A] table behind it.  One warp per row, one lane per position.
template <bool SCORES>
__global__ void __launch_bounds__(256) rows_pwm_generic_kernel(const uint8_t *base, const int64_t *starts, const int32_t *lens,
                                                               size_t n_rows, const uint8_t *lut, int alphabet_size,
                                                               const double *matrix, int m, int tail, const int64_t *offsets,
                                                               double *out, int64_t *status) {
    extern __shared__ __align__(16) uint32_t smem[];
    double *s_tab = reinterpret_cast<double *>(smem);
    uint8_t *s_lut = reinterpret_cast<uint8_t *>(s_tab + alphabet_size * m);
    const int tid = threadIdx.x, lane = tid & 31;
    s_lut[tid] = lut ? lut[tid] : (tid < alphabet_size ? (uint8_t)tid : (uint8_t)255);
    for (int i = tid; i < alphabet_size * m; i += 256) s_tab[i] = matrix[i];
    __syncthreads();
    uint64_t acc_values = 0, acc_bases = 0;
    const size_t warp_global = ((size_t)blockIdx.x * blockDim.x + tid) >> 5;
    const size_t n_warps = ((size_t)gridDim.x * blockDim.x) >> 5;
    for (size_t r = warp_global; r < n_rows; r += n_warps) {
        const uint8_t *row = base + starts[r];
        const int64_t L = lens[r];
        double best = -INFINITY;
        if (L > 0) {
            if (lane == 0) acc_bases += (uint64_t)L;
            int64_t first_bad = INT64_MAX;                  // every byte is validated, as the reference encodes it all
            for (int64_t i = lane; i < L; i += 32)
                if (s_lut[row[i]] >= alphabet_size) { first_bad = i; break; }
#pragma unroll
            for (int o = 16; o; o >>= 1) first_bad = min(first_bad, __shfl_xor_sync(0xffffffffu, first_bad, o));
            if (lane == 0 && first_bad != INT64_MAX)
                report_fault(status, fault_row_pos(r, first_bad));
            const int64_t npos = tail ? L : L - m + 1;
            double *o_row = SCORES ? out + offsets[r] : nullptr;
            for (int64_t i = lane; i < npos; i += 32) {
                const int nc = (int)min((int64_t)m, L - i);
                double s = 0.0;
                for (int j = 0; j < nc; ++j) {
                    const uint32_t c = s_lut[row[i + j]];
                    s += s_tab[j * alphabet_size + (c < (uint32_t)alphabet_size ? c : 0u)];
                }
                if constexpr (SCORES) o_row[i] = s;
                else best = nan_max(best, s);
                ++acc_values;
            }
        }
        if constexpr (!SCORES) {
#pragma unroll
            for (int o = 16; o; o >>= 1) best = nan_max(best, __shfl_xor_sync(0xffffffffu, best, o));
            if (lane == 0) out[r] = best;
        }
    }
    acc_values = warp_sum_u64(acc_values);
    acc_bases = warp_sum_u64(acc_bases);
    if (lane == 0) {
        if (acc_values) atomicAdd((unsigned long long *)&status[BNPK_ST_N_VALUES], acc_values);
        if (acc_bases) atomicAdd((unsigned long long *)&status[BNPK_ST_N_BASES], acc_bases);
    }
}

// Matches for alphabets that are not four letters (amino acids, "ACGTN") and raw bytes (alphabet_size 256): the same
// positions, sub-patterns and "same" tail as rows_match_kernel, with codes from a 256-byte LUT in shared memory
// (255 = invalid; byte codes: c < A maps to itself; raw bytes: every byte is its own code) and the column sets behind
// the sub-pattern table.  One warp per row, one lane per position; a sub-pattern stops at its first failed column.
// Writes out[offsets[r] + i] = 0/1 (OUT) or out[r] = the row's matches (int64).
template <bool OUT>
__global__ void __launch_bounds__(256) rows_match_generic_kernel(const uint8_t *base, const int64_t *starts,
                                                                 const int32_t *lens, size_t n_rows, const uint8_t *lut,
                                                                 int alphabet_size, const __grid_constant__ MatchArgs m,
                                                                 const int64_t *offsets, void *out, int64_t *status) {
    extern __shared__ __align__(16) uint32_t smem[];
    int *s_len = reinterpret_cast<int *>(smem);
    int *s_col = s_len + kMatchMaxSubs;
    uint32_t *s_sets = reinterpret_cast<uint32_t *>(s_col + kMatchMaxSubs);
    uint8_t *s_lut = reinterpret_cast<uint8_t *>(s_sets + m.n_words);
    const int tid = threadIdx.x, lane = tid & 31;
    const uint32_t A = (uint32_t)alphabet_size, wpc = (uint32_t)m.words_per_col;
    s_lut[tid] = lut ? lut[tid] : ((uint32_t)tid < A ? (uint8_t)tid : (uint8_t)255);
    if (tid == 0) {
        int col = 0;
#pragma unroll
        for (int k = 0; k < kMatchMaxSubs; ++k)
            if (k < m.n_sub) { s_len[k] = m.len[k]; s_col[k] = col; col += m.len[k]; }
    }
    for (int i = tid; i < m.n_words; i += 256) s_sets[i] = m.sets[i];
    __syncthreads();
    uint64_t acc_values = 0, acc_bases = 0;
    const size_t warp_global = ((size_t)blockIdx.x * blockDim.x + tid) >> 5;
    const size_t n_warps = ((size_t)gridDim.x * blockDim.x) >> 5;
    for (size_t r = warp_global; r < n_rows; r += n_warps) {
        const uint8_t *row = base + starts[r];
        const int64_t L = lens[r];
        uint64_t hits = 0;
        if (L > 0) {
            if (lane == 0) acc_bases += (uint64_t)L;
            if (A < 256) {                                  // every byte is validated, as the reference encodes it all
                int64_t first_bad = INT64_MAX;
                for (int64_t i = lane; i < L; i += 32)
                    if (s_lut[row[i]] >= A) { first_bad = i; break; }
#pragma unroll
                for (int o = 16; o; o >>= 1) first_bad = min(first_bad, __shfl_xor_sync(0xffffffffu, first_bad, o));
                if (lane == 0 && first_bad != INT64_MAX)
                    report_fault(status, fault_row_pos(r, first_bad));
            }
            const int64_t npos = m.same ? L : L - m.span + 1;
            uint8_t *o_row = OUT ? reinterpret_cast<uint8_t *>(out) + offsets[r] : nullptr;
            for (int64_t i = lane; i < npos; i += 32) {
                bool hit = false;
                for (int k = 0; k < m.n_sub && !hit; ++k) {
                    const int mk = s_len[k];
                    if (i + mk > L) continue;
                    const uint32_t *set = s_sets + (size_t)s_col[k] * wpc;
                    bool ok = true;
                    for (int j = 0; j < mk && ok; ++j) {
                        const uint32_t c = s_lut[row[i + j]];
                        ok = c < A && ((set[j * wpc + (c >> 5)] >> (c & 31u)) & 1u);
                    }
                    hit = ok;
                }
                if constexpr (OUT) o_row[i] = (uint8_t)hit;
                hits += hit;
                ++acc_values;
            }
        }
        if constexpr (!OUT) {
            hits = warp_sum_u64(hits);
            if (lane == 0) reinterpret_cast<int64_t *>(out)[r] = (int64_t)hits;
        }
    }
    acc_values = warp_sum_u64(acc_values);
    acc_bases = warp_sum_u64(acc_bases);
    if (lane == 0) {
        if (acc_values) atomicAdd((unsigned long long *)&status[BNPK_ST_N_VALUES], acc_values);
        if (acc_bases) atomicAdd((unsigned long long *)&status[BNPK_ST_N_BASES], acc_bases);
    }
}

// get_reverse_complement (sequence/dna.py:36-65): out row r = lut[row r read backwards]; one warp per row,
// coalesced writes.  The 256-byte lut is the reference's complement Lookup for the array's encoding.
__global__ void __launch_bounds__(256) rows_reverse_complement_kernel(const uint8_t *base, const int64_t *starts, const int32_t *lens,
                                                                      size_t n_rows, const uint8_t *lut, const int64_t *offsets,
                                                                      uint8_t *out) {
    __shared__ uint8_t s_lut[256];
    const int tid = threadIdx.x, lane = tid & 31;
    s_lut[tid] = lut[tid];
    __syncthreads();
    const size_t warp_global = ((size_t)blockIdx.x * blockDim.x + tid) >> 5;
    const size_t n_warps = ((size_t)gridDim.x * blockDim.x) >> 5;
    for (size_t r = warp_global; r < n_rows; r += n_warps) {
        const int64_t start = starts[r], L = lens[r], o = offsets[r];
        for (int64_t i = lane; i < L; i += 32) out[o + i] = s_lut[base[start + L - 1 - i]];
    }
}

static size_t rows_smem_bytes(bool counting, bool smem_hist, uint64_t n_bins) {
    size_t b = (size_t)kRowWarps * kWarpWords * 4 + 256;
    if (counting && smem_hist) b += n_bins * 4;
    return b;
}

static const char *const kRowsMisfit = "rows kernel does not fit shared memory";

template <int RM, int ENC, bool SMEM_HIST, bool DEFERRED>
static int launch_rows_t(const RowArgs &a, size_t est_rows, cudaStream_t st) {
    constexpr bool PWM = (RM == RM_PWM || RM == RM_PWM_MAX);
    void (*kern)(const RowArgs);
    if constexpr (PWM) kern = rows_pwm_kernel<RM, ENC>;
    else kern = rows_kernel<RM, ENC, SMEM_HIST, DEFERRED>;
    constexpr bool COUNTING = (RM == RM_COUNT || RM == RM_COUNT_MIN);
    size_t smem = rows_smem_bytes(COUNTING, SMEM_HIST, a.n_bins);
    if constexpr (PWM) smem += (size_t)4 * a.window * sizeof(double);
    return launch_resident(PWM ? "rows_pwm_kernel" : "rows_kernel", kRowsMisfit, kern, (est_rows + kRowWarps - 1) / kRowWarps,
                           kRowThreads, smem, 200 * 1024, st, false, a);
}

template <int RM, bool SMEM_HIST, bool DEFERRED>
static int launch_rows_enc(const RowArgs &a, int enc_mode, size_t est_rows, cudaStream_t st) {
    return with_enc(enc_mode, [&](auto enc) {
        return launch_rows_t<RM, decltype(enc)::value, SMEM_HIST, DEFERRED>(a, est_rows, st);
    });
}

// The kernels' view of a row entry point's rows (n_bins 1 for the modes that count nothing); the caller fills in its
// mode's fields.
static RowArgs row_args(const uint8_t *base, size_t base_bytes, const int64_t *starts, const int32_t *lens,
                        size_t n_rows, const uint8_t *lut256) {
    RowArgs a{};
    a.base = base; a.base_bytes = base_bytes; a.starts = starts; a.lens = lens; a.n_rows = n_rows; a.lut = lut256;
    a.n_bins = 1;
    return a;
}

static int check_common(int enc_mode, const uint8_t *lut256, int k, int window) {
    if (k < 1 || k > 31) return set_err(BNPK_E_K, "k must be larger than 0 and smaller than 32");
    if (window != 0 && window < k) return set_err(BNPK_E_WINDOW, "kmer size must be smaller than window size");
    if (window > kSegBytes / 2) return set_err(BNPK_E_WINDOW, "window_size above 1024 is not supported");
    return check_enc(enc_mode, lut256, 4);
}

template <bool MINZ>
static int launch_uncount(const RowArgs &a, int enc_mode, cudaStream_t st) {
    return with_enc(enc_mode, [&](auto enc) {
        return launch("uncount_kernel", uncount_kernel<decltype(enc)::value, MINZ>, 1, 32, kWarpWords * 4 + 256, st,
                      false, a);
    });
}

int count_fixups_impl(const uint8_t *chunk, size_t n, int lpe, int enc_mode, const uint8_t *lut256, int k,
                      int window, int64_t n_bins, int64_t *hist, int64_t *status, const uint64_t *deferred_count,
                      const uint64_t *deferred, size_t deferred_cap, cudaStream_t st) {
    RowArgs a{};
    a.base = chunk; a.base_bytes = n; a.lut = lut256; a.k = k; a.window = window;
    a.n_bins = (uint64_t)n_bins; a.hist = (unsigned long long *)hist; a.status = status;
    a.deferred_count = deferred_count; a.deferred = deferred; a.deferred_cap = deferred_cap; a.lpe = lpe;
    // long rows: a modest fixed grid; the kernel reads the row count on the device
    const size_t est = (size_t)sm_count() * kRowWarps * 2;
    int rc = window ? launch_rows_enc<RM_COUNT_MIN, false, true>(a, enc_mode, est, st)
                    : launch_rows_enc<RM_COUNT, false, true>(a, enc_mode, est, st);
    if (rc) return rc;
    return window ? launch_uncount<true>(a, enc_mode, st) : launch_uncount<false>(a, enc_mode, st);
}

static int check_pwm(int enc_mode, const uint8_t *lut256, int alphabet_size, const double *matrix, int motif_len) {
    if (motif_len < 1 || motif_len > kPwmMaxLen) return set_err(BNPK_E_BADARG, "motif_len must be in 1..1024");
    if (alphabet_size < 2 || alphabet_size > 255) return set_err(BNPK_E_BADARG, "alphabet_size must be in 2..255");
    if (alphabet_size * motif_len > kPwmMaxCells) return set_err(BNPK_E_BADARG, "alphabet_size * motif_len above 8192");
    if (int rc = check_enc(enc_mode, lut256, alphabet_size)) return rc;
    if (!matrix) return set_err(BNPK_E_BADARG, "matrix required");
    return 0;
}

// Four-letter alphabets take rows_kernel's motif modes (2-bit codes, every enc_mode); the others the byte-LUT kernel.
template <bool SCORES>
static int launch_pwm(const uint8_t *base, size_t base_bytes, const int64_t *starts, const int32_t *lens, size_t n_rows,
                      int enc_mode, const uint8_t *lut256, int alphabet_size, const double *matrix, int motif_len,
                      int tail, const int64_t *offsets, double *out, int64_t *status, cudaStream_t st) {
    if (alphabet_size == 4) {
        RowArgs a = row_args(base, base_bytes, starts, lens, n_rows, lut256);
        a.k = 1; a.window = motif_len; a.offsets = offsets; a.out = out; a.status = status;
        a.pwm = matrix; a.tail = tail;
        return launch_rows_enc<SCORES ? RM_PWM : RM_PWM_MAX, false, false>(a, enc_mode, n_rows, st);
    }
    auto kern = rows_pwm_generic_kernel<SCORES>;
    const size_t smem = (size_t)alphabet_size * motif_len * sizeof(double) + 256;
    BNPK_DYN_SMEM(kern, kPwmMaxCells * sizeof(double) + 256);
    return launch("rows_pwm_generic_kernel", kern, grid_cap((n_rows + 7) / 8, 8), 256, smem, st, false, base, starts,
                  lens, n_rows, enc_mode == BNPK_ENC_LUT ? lut256 : nullptr, alphabet_size, matrix, motif_len, tail,
                  offsets, out, status);
}

// The limits of bnpk_rows_match*, and the kernels' view of the pattern in `m`.
static int check_match(int enc_mode, const uint8_t *lut256, int alphabet_size, const uint32_t *sets,
                       const int32_t *sub_lens, int n_sub, int same, MatchArgs &m) {
    if (alphabet_size < 2 || alphabet_size > 256) return set_err(BNPK_E_BADARG, "alphabet_size must be in 2..256");
    if (int rc = check_enc(enc_mode, lut256, alphabet_size)) return rc;
    if (!sets || !sub_lens) return set_err(BNPK_E_BADARG, "sets and sub_lens required");
    if (n_sub < 1 || n_sub > kMatchMaxSubs) return set_err(BNPK_E_BADARG, "n_sub must be in 1..64");
    if (same != 0 && same != 1) return set_err(BNPK_E_BADARG, "same must be 0 or 1");
    m = MatchArgs{};
    m.sets = sets; m.n_sub = n_sub; m.same = same; m.words_per_col = (alphabet_size + 31) / 32;
    int cols = 0;
    for (int k = 0; k < n_sub; ++k) {
        if (sub_lens[k] < 1 || sub_lens[k] > kMatchMaxLen) return set_err(BNPK_E_BADARG, "sub-pattern lengths must be in 1..1024");
        m.len[k] = sub_lens[k];
        m.span = std::max(m.span, (int)sub_lens[k]);
        cols += sub_lens[k];
    }
    if ((int64_t)cols * m.words_per_col > kMatchMaxWords)
        return set_err(BNPK_E_BADARG, "symbol sets above 8192 words (columns * ceil(alphabet_size / 32))");
    m.n_words = cols * m.words_per_col;
    return 0;
}

// Four-letter alphabets take rows_match_kernel (2-bit codes, every enc_mode); the others and raw bytes the LUT kernel.
template <bool OUT>
static int launch_match(const uint8_t *base, size_t base_bytes, const int64_t *starts, const int32_t *lens,
                        size_t n_rows, int enc_mode, const uint8_t *lut256, int alphabet_size, const MatchArgs &m,
                        const int64_t *offsets, void *out, int64_t *status, cudaStream_t st) {
    constexpr int RM = OUT ? RM_MATCH : RM_MATCH_COUNT;
    if (alphabet_size == 4) {
        RowArgs a = row_args(base, base_bytes, starts, lens, n_rows, lut256);
        a.k = 1; a.window = m.span; a.offsets = offsets; a.out = out; a.status = status;
        const size_t smem_head = rows_smem_bytes(false, false, 0) + kMatchSmemHead;
        return with_enc(enc_mode, [&](auto enc) {
            return launch_resident("rows_match_kernel", kRowsMisfit, rows_match_kernel<RM, decltype(enc)::value>,
                                   (n_rows + kRowWarps - 1) / kRowWarps, kRowThreads, smem_head + (size_t)m.n_words * 4,
                                   smem_head + kMatchMaxWords * 4, st, false, a, m);
        });
    }
    auto kern = rows_match_generic_kernel<OUT>;
    const size_t smem = kMatchSmemHead + (size_t)m.n_words * 4 + 256;
    BNPK_DYN_SMEM(kern, kMatchSmemHead + kMatchMaxWords * 4 + 256);
    return launch("rows_match_generic_kernel", kern, grid_cap((n_rows + 7) / 8, 8), 256, smem, st, false, base,
                  starts, lens, n_rows, enc_mode == BNPK_ENC_LUT ? lut256 : nullptr, alphabet_size, m, offsets, out,
                  status);
}

static uint64_t canon_pattern(int complement_xor) {
    return complement_xor == 3 ? ~0ull : complement_xor == 2 ? 0xAAAAAAAAAAAAAAAAull : 0x5555555555555555ull;
}

static int check_canonical(bool canonical, int complement_xor) {
    if (canonical && (complement_xor < 1 || complement_xor > 3))
        return set_err(BNPK_E_BADARG, "complement_xor must be 1, 2 or 3");
    return 0;
}

// bnpk_rows_kmer_hash, bnpk_rows_kmer_hash_canonical and bnpk_rows_minimizers: the k-mer hashes of every row
// (canonical ones with `canonical`), or their minima over every window of `window` bases.
static int rows_kmer_hash(const uint8_t *base, size_t base_bytes, const int64_t *starts, const int32_t *lens,
                          size_t n_rows, int enc_mode, const uint8_t *lut256, int k, int window, bool canonical,
                          int complement_xor, const int64_t *offsets, int64_t *out, int64_t *status, void *stream) {
    if (int rc = check_common(enc_mode, lut256, k, window)) return rc;
    if (int rc = check_canonical(canonical, complement_xor)) return rc;
    if (n_rows == 0) return 0;
    RowArgs a = row_args(base, base_bytes, starts, lens, n_rows, lut256);
    a.k = k; a.window = window; a.offsets = offsets; a.out = out; a.status = status;
    if (canonical) a.canon_xor = canon_pattern(complement_xor);
    cudaStream_t st = (cudaStream_t)stream;
    return window ? launch_rows_enc<RM_MINIMIZER, false, false>(a, enc_mode, n_rows, st)
                  : launch_rows_enc<RM_HASH, false, false>(a, enc_mode, n_rows, st);
}

// bnpk_rows_kmer_count and bnpk_rows_kmer_count_canonical: the k-mers of every row (canonical ones with `canonical`),
// or their window minima, counted into hist.
static int rows_kmer_count(const uint8_t *base, size_t base_bytes, const int64_t *starts, const int32_t *lens,
                           size_t n_rows, int enc_mode, const uint8_t *lut256, int k, int window, bool canonical,
                           int complement_xor, int64_t n_bins, int hist_mode, int64_t *hist, int64_t *status,
                           void *stream) {
    if (int rc = check_common(enc_mode, lut256, k, window)) return rc;
    if (int rc = check_canonical(canonical, complement_xor)) return rc;
    if (n_bins < 1) return set_err(BNPK_E_BINS, "n_bins must be positive");
    if (hist_mode == BNPK_HIST_SMEM && n_bins > kSmemMaxBins) return set_err(BNPK_E_BINS, "too many bins for the shared-memory histogram");
    if (n_rows == 0) return 0;
    RowArgs a = row_args(base, base_bytes, starts, lens, n_rows, lut256);
    a.k = k; a.window = window; a.n_bins = (uint64_t)n_bins; a.hist = (unsigned long long *)hist; a.status = status;
    if (canonical) a.canon_xor = canon_pattern(complement_xor);
    const bool sm = use_smem_hist(n_bins, hist_mode);
    cudaStream_t st = (cudaStream_t)stream;
    if (window)
        return sm ? launch_rows_enc<RM_COUNT_MIN, true, false>(a, enc_mode, n_rows, st)
                  : launch_rows_enc<RM_COUNT_MIN, false, false>(a, enc_mode, n_rows, st);
    return sm ? launch_rows_enc<RM_COUNT, true, false>(a, enc_mode, n_rows, st)
              : launch_rows_enc<RM_COUNT, false, false>(a, enc_mode, n_rows, st);
}

}  // namespace bnpk

using namespace bnpk;

extern "C" {

int bnpk_rows_encode(const uint8_t *base, size_t base_bytes, const int64_t *starts, const int32_t *lens, size_t n_rows,
                     int enc_mode, const uint8_t *lut256, const int64_t *offsets, uint8_t *codes_out,
                     int64_t *status, void *stream) {
    if (int rc = check_common(enc_mode, lut256, 1, 0)) return rc;
    if (n_rows == 0) return 0;
    RowArgs a = row_args(base, base_bytes, starts, lens, n_rows, lut256);
    a.k = 1; a.offsets = offsets; a.out = codes_out; a.status = status;
    return launch_rows_enc<RM_ENCODE, false, false>(a, enc_mode, n_rows, (cudaStream_t)stream);
}

int bnpk_rows_kmer_hash(const uint8_t *base, size_t base_bytes, const int64_t *starts, const int32_t *lens, size_t n_rows,
                        int enc_mode, const uint8_t *lut256, int k, const int64_t *offsets, int64_t *hashes_out,
                        int64_t *status, void *stream) {
    return rows_kmer_hash(base, base_bytes, starts, lens, n_rows, enc_mode, lut256, k, 0, false, 0, offsets, hashes_out,
                          status, stream);
}

int bnpk_rows_generic_hash(const uint8_t *base, size_t base_bytes, const int64_t *starts, const int32_t *lens, size_t n_rows,
                            const uint8_t *lut256, int alphabet_size, int k, const int64_t *offsets, int64_t *hashes_out,
                            int64_t *status, void *stream) {
    if (k < 1 || k > 63) return set_err(BNPK_E_K, "k must be in 1..63 for the generic hash");
    if (alphabet_size < 2 || alphabet_size > 255) return set_err(BNPK_E_BADARG, "alphabet_size must be in 2..255");
    if (n_rows == 0) return 0;
    return launch("rows_generic_hash_kernel", rows_generic_hash_kernel, grid_cap((n_rows + 7) / 8, 8), 256, 0,
                  (cudaStream_t)stream, false, base, base_bytes, starts, lens, n_rows, lut256, alphabet_size, k,
                  offsets, hashes_out, status);
}

int bnpk_rows_minimizers(const uint8_t *base, size_t base_bytes, const int64_t *starts, const int32_t *lens, size_t n_rows,
                         int enc_mode, const uint8_t *lut256, int k, int window_size, const int64_t *offsets,
                         int64_t *mins_out, int64_t *status, void *stream) {
    if (window_size < 1) return set_err(BNPK_E_WINDOW, "window_size must be positive");
    return rows_kmer_hash(base, base_bytes, starts, lens, n_rows, enc_mode, lut256, k, window_size, false, 0, offsets,
                          mins_out, status, stream);
}

int bnpk_rows_kmer_count(const uint8_t *base, size_t base_bytes, const int64_t *starts, const int32_t *lens, size_t n_rows,
                         int enc_mode, const uint8_t *lut256, int k, int window_size, int64_t n_bins, int hist_mode,
                         int64_t *hist, int64_t *status, void *stream) {
    return rows_kmer_count(base, base_bytes, starts, lens, n_rows, enc_mode, lut256, k, window_size, false, 0, n_bins,
                           hist_mode, hist, status, stream);
}

int bnpk_rows_kmer_hash_canonical(const uint8_t *base, size_t base_bytes, const int64_t *starts, const int32_t *lens,
                                  size_t n_rows, int enc_mode, const uint8_t *lut256, int k, int complement_xor,
                                  const int64_t *offsets, int64_t *hashes_out, int64_t *status, void *stream) {
    return rows_kmer_hash(base, base_bytes, starts, lens, n_rows, enc_mode, lut256, k, 0, true, complement_xor, offsets,
                          hashes_out, status, stream);
}

int bnpk_rows_kmer_count_canonical(const uint8_t *base, size_t base_bytes, const int64_t *starts, const int32_t *lens,
                                   size_t n_rows, int enc_mode, const uint8_t *lut256, int k, int complement_xor,
                                   int64_t n_bins, int hist_mode, int64_t *hist, int64_t *status, void *stream) {
    return rows_kmer_count(base, base_bytes, starts, lens, n_rows, enc_mode, lut256, k, 0, true, complement_xor, n_bins,
                           hist_mode, hist, status, stream);
}

static bool is_pow2(size_t c) { return c && (c & (c - 1)) == 0; }

int bnpk_rows_kmer_table_insert(const uint8_t *base, size_t base_bytes, const int64_t *starts, const int32_t *lens,
                                size_t n_rows, int enc_mode, const uint8_t *lut256, int k, int complement_xor,
                                int64_t *keys, int64_t *counts, size_t capacity, int64_t *n_used,
                                int64_t *status, void *stream) {
    if (int rc = check_common(enc_mode, lut256, k, 0)) return rc;
    if (complement_xor < 0 || complement_xor > 3) return set_err(BNPK_E_BADARG, "complement_xor must be 0, 1, 2 or 3");
    if (!is_pow2(capacity)) return set_err(BNPK_E_BADARG, "table capacity must be a power of two");
    if (n_rows == 0) return 0;
    RowArgs a = row_args(base, base_bytes, starts, lens, n_rows, lut256);
    a.k = k; a.status = status;
    a.canon_xor = complement_xor ? canon_pattern(complement_xor) : 0;
    a.table.keys = (unsigned long long *)keys; a.table.counts = (unsigned long long *)counts;
    a.table.mask = capacity - 1; a.table.n_used = (unsigned long long *)n_used;
    return launch_rows_enc<RM_TABLE, false, false>(a, enc_mode, n_rows, (cudaStream_t)stream);
}

int bnpk_kmer_table_rehash(const int64_t *keys, const int64_t *counts, size_t capacity,
                           int64_t *new_keys, int64_t *new_counts, size_t new_capacity, int64_t *n_used,
                           int64_t *status, void *stream) {
    if (!is_pow2(capacity) || !is_pow2(new_capacity)) return set_err(BNPK_E_BADARG, "table capacity must be a power of two");
    KmerTable t;
    t.keys = (unsigned long long *)new_keys; t.counts = (unsigned long long *)new_counts;
    t.mask = new_capacity - 1; t.n_used = (unsigned long long *)n_used;
    return launch("table_rehash_kernel", table_rehash_kernel, grid_cap((capacity + 255) / 256, 8), 256, 0,
                  (cudaStream_t)stream, false, keys, counts, capacity, t, status);
}

int bnpk_rows_reverse_complement(const uint8_t *base, size_t base_bytes, const int64_t *starts, const int32_t *lens,
                                 size_t n_rows, const uint8_t *lut256, const int64_t *offsets, uint8_t *out, void *stream) {
    (void)base_bytes;
    if (!lut256) return set_err(BNPK_E_BADARG, "lut256 required");
    if (n_rows == 0) return 0;
    return launch("rows_reverse_complement_kernel", rows_reverse_complement_kernel, grid_cap((n_rows + 7) / 8, 8), 256,
                  0, (cudaStream_t)stream, false, base, starts, lens, n_rows, lut256, offsets, out);
}

int bnpk_rows_pwm_scores(const uint8_t *base, size_t base_bytes, const int64_t *starts, const int32_t *lens,
                         size_t n_rows, int enc_mode, const uint8_t *lut256, int alphabet_size,
                         const double *matrix, int motif_len, int tail,
                         const int64_t *offsets, double *scores_out, int64_t *status, void *stream) {
    if (int rc = check_pwm(enc_mode, lut256, alphabet_size, matrix, motif_len)) return rc;
    if (tail != 0 && tail != 1) return set_err(BNPK_E_BADARG, "tail must be 0 or 1");
    if (n_rows == 0) return 0;
    return launch_pwm<true>(base, base_bytes, starts, lens, n_rows, enc_mode, lut256, alphabet_size, matrix, motif_len,
                            tail, offsets, scores_out, status, (cudaStream_t)stream);
}

int bnpk_rows_pwm_max(const uint8_t *base, size_t base_bytes, const int64_t *starts, const int32_t *lens,
                      size_t n_rows, int enc_mode, const uint8_t *lut256, int alphabet_size,
                      const double *matrix, int motif_len, double *max_out, int64_t *status, void *stream) {
    if (int rc = check_pwm(enc_mode, lut256, alphabet_size, matrix, motif_len)) return rc;
    if (n_rows == 0) return 0;
    return launch_pwm<false>(base, base_bytes, starts, lens, n_rows, enc_mode, lut256, alphabet_size, matrix, motif_len,
                             0, nullptr, max_out, status, (cudaStream_t)stream);
}

int bnpk_rows_match(const uint8_t *base, size_t base_bytes, const int64_t *starts, const int32_t *lens, size_t n_rows,
                    int enc_mode, const uint8_t *lut256, int alphabet_size, const uint32_t *sets,
                    const int32_t *sub_lens, int n_sub, int same, const int64_t *offsets, uint8_t *match_out,
                    int64_t *status, void *stream) {
    MatchArgs m;
    if (int rc = check_match(enc_mode, lut256, alphabet_size, sets, sub_lens, n_sub, same, m)) return rc;
    if (n_rows == 0) return 0;
    return launch_match<true>(base, base_bytes, starts, lens, n_rows, enc_mode, lut256, alphabet_size, m, offsets,
                              match_out, status, (cudaStream_t)stream);
}

int bnpk_rows_match_count(const uint8_t *base, size_t base_bytes, const int64_t *starts, const int32_t *lens,
                          size_t n_rows, int enc_mode, const uint8_t *lut256, int alphabet_size, const uint32_t *sets,
                          const int32_t *sub_lens, int n_sub, int same, int64_t *count_out, int64_t *status,
                          void *stream) {
    MatchArgs m;
    if (int rc = check_match(enc_mode, lut256, alphabet_size, sets, sub_lens, n_sub, same, m)) return rc;
    if (n_rows == 0) return 0;
    return launch_match<false>(base, base_bytes, starts, lens, n_rows, enc_mode, lut256, alphabet_size, m, nullptr,
                               count_out, status, (cudaStream_t)stream);
}

}  // extern "C"
