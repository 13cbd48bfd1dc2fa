// write_kernels.cu -- records -> file text on the device: FASTQ, two-line FASTA and wrapped FASTA
// (FastQBuffer.from_data / join_fields io/fastq_buffer.py:47-61, OneLineBuffer.join_fields io/one_line_buffer.py:119-134,
// MultiLineFastaBuffer.from_data io/multiline_buffer.py:67-86).
//
// Entry e with name, sequence and quality lengths Ln, Ls, Lq is laid out as
//   FASTQ          '@' name '\n' seq '\n' '+' '\n' qual '\n'                     Ln + Ls + Lq + 6 bytes
//   two-line FASTA '>' name '\n' seq '\n'                                        Ln + Ls + 3
//   wrapped FASTA  '>' name '\n', then ceil(Ls / W) lines of W bases (the last one shorter), each ending in '\n'
//                                                                                Ln + 2 + Ls + ceil(Ls / W)
// format_offsets_kernel is the exclusive prefix sum of those sizes (the single-pass scan of bnpk_device.cuh, as bnpk_row_offsets).
// format_kernel is output-driven: a CTA owns a tile of output bytes, finds the entry of each 16-byte unit by a binary
// search of the offsets and builds the unit in registers -- one unaligned 16-byte gather when the unit lies inside one
// field segment, byte by byte otherwise -- and writes it with one vector store.  The same kernel in CHECK mode walks
// the whole text without writing it and reports the first sequence byte whose LUT entry is 0.
//
// Delimited lines (BED, bedGraph; dump_csv io/dump_csv.py, join_columns io/strops.py:186-215): line e is its columns
// joined by '\t' and ended by '\n'.  delimited_offsets_kernel is the exclusive prefix sum of the line sizes;
// delimited_text_kernel is output-driven: a CTA owns a 16 KiB window of output, finds its lines by a binary search of
// the offsets, builds them one line per thread in shared memory and stores the window with 16-byte stores.
#include "bnpk_host.h"

namespace bnpk {

namespace {

constexpr int kFmtThreads = 256;
constexpr int kFmtUnitsPerThread = 4;
constexpr int64_t kFmtTile = (int64_t)kFmtThreads * kFmtUnitsPerThread * 16;   // 16 KiB of output per tile

struct FmtArgs {
    const uint8_t *base[3];
    uint64_t base_bytes[3];
    const int64_t *starts[3];
    const int32_t *lens[3];
    const uint8_t *lut[3];
    int fmt;
    int width;
    int64_t n;                  // entries
    const int64_t *offs;        // int64[n + 1]
    int64_t out_begin, out_end; // CHECK: out_end < 0 means offs[n]
    uint8_t *out;
    int64_t *status;
};

__device__ __forceinline__ int64_t len_of(const int32_t *lens, int64_t e) {
    return lens ? (int64_t)max(lens[e], 0) : 0;
}

__device__ __forceinline__ int64_t entry_size(int fmt, int width, int64_t ln, int64_t ls, int64_t lq) {
    if (fmt == BNPK_FMT_FASTQ) return ln + ls + lq + 6;
    if (fmt == BNPK_FMT_FASTA) return ln + ls + 3;
    return ln + 2 + ls + (ls + width - 1) / width;
}

// exclusive prefix sum of the entry sizes; offs[n] = total
__global__ void __launch_bounds__(kScanThreads) format_offsets_kernel(const __grid_constant__ FmtArgs a, int64_t *offs,
                                                                      uint64_t *ws) {
    exclusive_offsets(a.n, offs, ws, [&](int64_t e) -> uint64_t {
        return (uint64_t)entry_size(a.fmt, a.width, len_of(a.lens[0], e), len_of(a.lens[1], e), len_of(a.lens[2], e));
    });
}

// the entry that holds output byte p: offs[e] <= p < offs[e + 1], searched in [lo, hi]
__device__ __forceinline__ int64_t find_entry(const int64_t *offs, int64_t lo, int64_t hi, int64_t p) {
    while (lo < hi) {
        const int64_t mid = (lo + hi + 1) >> 1;
        if (offs[mid] <= p) lo = mid;
        else hi = mid - 1;
    }
    return lo;
}

// one entry's view; the fields are named, not an array, so that picking one by a run-time index needs no stack
struct Entry {
    int64_t e, begin, end;      // output bytes [begin, end)
    int64_t s0, s1, s2;         // field starts
    int64_t l0, l1, l2;         // field lengths
    __device__ __forceinline__ int64_t start(int f) const { return f == 0 ? s0 : f == 1 ? s1 : s2; }
};

__device__ __forceinline__ int64_t start_of(const FmtArgs &a, int f, int64_t e, int64_t len) {
    return a.starts[f] && len ? a.starts[f][e] : 0;
}

__device__ __forceinline__ void load_entry(const FmtArgs &a, int64_t e, Entry &E) {
    E.e = e;
    E.begin = a.offs[e];
    E.end = a.offs[e + 1];
    E.l0 = len_of(a.lens[0], e);
    E.l1 = len_of(a.lens[1], e);
    E.l2 = len_of(a.lens[2], e);
    E.s0 = start_of(a, 0, e, E.l0);
    E.s1 = start_of(a, 1, e, E.l1);
    E.s2 = start_of(a, 2, e, E.l2);
}

// Where entry-relative byte q comes from: a constant byte (field < 0) or byte `idx` of field `field`.
struct Src {
    int field;
    int64_t idx;
    uint8_t c;
};

__device__ __forceinline__ Src locate(const FmtArgs &a, const Entry &E, int64_t q) {
    const int64_t ln = E.l0, ls = E.l1;
    if (q == 0) return {-1, 0, (uint8_t)(a.fmt == BNPK_FMT_FASTQ ? '@' : '>')};
    q -= 1;
    if (q < ln) return {0, q, 0};
    q -= ln;
    if (q == 0) return {-1, 0, '\n'};
    q -= 1;
    if (a.fmt == BNPK_FMT_FASTA_WRAPPED) {
        const int64_t w = a.width, line = q / (w + 1), col = q - line * (w + 1), idx = line * w + col;
        if (col == w || idx >= ls) return {-1, 0, '\n'};
        return {1, idx, 0};
    }
    if (q < ls) return {1, q, 0};
    q -= ls;
    if (a.fmt == BNPK_FMT_FASTA) return {-1, 0, '\n'};
    if (q < 3) return {-1, 0, (uint8_t)(q == 1 ? '+' : '\n')};
    q -= 3;
    if (q < E.l2) return {2, q, 0};
    return {-1, 0, '\n'};
}

// A unit [q, q + 16) of the entry that lies inside one field segment: (field, first index), else field -1.
__device__ __forceinline__ Src whole_unit(const FmtArgs &a, const Entry &E, int64_t q) {
    const int64_t ln = E.l0, ls = E.l1;
    if (q >= 1 && q + 16 <= 1 + ln) return {0, q - 1, 0};
    const int64_t s0 = 2 + ln;
    if (a.fmt == BNPK_FMT_FASTA_WRAPPED) {
        const int64_t w = a.width;
        if (w >= 16 && q >= s0) {
            const int64_t r = q - s0, line = r / (w + 1), col = r - line * (w + 1), idx = line * w + col;
            if (col + 16 <= w && idx + 16 <= ls) return {1, idx, 0};
        }
        return {-1, 0, 0};
    }
    if (q >= s0 && q + 16 <= s0 + ls) return {1, q - s0, 0};
    if (a.fmt == BNPK_FMT_FASTQ) {
        const int64_t s2 = s0 + ls + 3;
        if (q >= s2 && q + 16 <= s2 + E.l2) return {2, q - s2, 0};
    }
    return {-1, 0, 0};
}

// bad bytes are the error path: each one goes straight to the status word
__device__ __forceinline__ void report_bad(int64_t *status, int64_t v) {
    atomicMin((long long *)&status[BNPK_ST_BAD_BASE], (long long)v);
}

template <bool CHECK>
__global__ void __launch_bounds__(kFmtThreads) format_kernel(const __grid_constant__ FmtArgs a) {
    __shared__ uint8_t s_lut[3][256];
    for (int i = threadIdx.x; i < 3 * 256; i += kFmtThreads) {
        const int f = i >> 8;
        s_lut[f][i & 255] = a.lut[f] ? a.lut[f][i & 255] : (uint8_t)(i & 255);
    }
    __syncthreads();
    const int64_t n = a.n;
    const int64_t begin = a.out_begin;
    const int64_t end = CHECK ? a.offs[n] : a.out_end;
    if (end <= begin) return;
    // out-relative units start where out + j is 16-byte aligned: a head unit of `head` bytes, then whole units
    const int head = CHECK ? 0 : (int)((16 - (reinterpret_cast<uintptr_t>(a.out) & 15)) & 15);
    const int64_t span = end - begin;
    const int64_t n_units = head ? 1 + (max(span - head, (int64_t)0) + 15) / 16 : (span + 15) / 16;
    constexpr int64_t kTileUnits = kFmtThreads * kFmtUnitsPerThread;
    const int64_t n_tiles = (n_units + kTileUnits - 1) / kTileUnits;
    // out-relative first byte of unit u
    auto unit_j0 = [head](int64_t u) -> int64_t { return head ? (u == 0 ? 0 : head + (u - 1) * 16) : u * 16; };
    for (int64_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
        const int64_t u_first = tile * kTileUnits;
        // entries of the tile: [lo, hi]
        const int64_t lo = find_entry(a.offs, 0, n - 1, begin + unit_j0(u_first));
        const int64_t hi = find_entry(a.offs, lo, n - 1, begin + min(span, unit_j0(u_first + kTileUnits)) - 1);
#pragma unroll 1
        for (int k = 0; k < kFmtUnitsPerThread; ++k) {
            const int64_t u = u_first + (int64_t)k * kFmtThreads + threadIdx.x;
            // out-relative byte range [j0, j1) of unit u
            const int64_t j0 = unit_j0(u);
            if (j0 >= span) break;
            const int64_t j1 = min(unit_j0(u + 1), span);
            const int64_t p0 = begin + j0;
            Entry E;
            load_entry(a, find_entry(a.offs, lo, hi, p0), E);
            uint32_t w[4] = {0u, 0u, 0u, 0u};
            const Src whole = (j1 - j0 == 16) ? whole_unit(a, E, p0 - E.begin) : Src{-1, 0, 0};
            bool fast = whole.field >= 0;
            if (fast) {
                const int f = whole.field;
                const int64_t src = E.start(f) + whole.idx;
                fast = src >= 0 && (uint64_t)(src + 16) <= a.base_bytes[f];
                if (fast && (!CHECK || f == 1)) {
                    load16(a.base[f] + src, w);
                    if (a.lut[f]) {
#pragma unroll
                        for (int i = 0; i < 4; ++i) {
                            uint32_t r = 0;
#pragma unroll
                            for (int b = 0; b < 4; ++b) {
                                const uint8_t c = s_lut[f][(w[i] >> (8 * b)) & 255];
                                if (CHECK && c == 0) report_bad(a.status, (E.e << 32) | (whole.idx + 4 * i + b));
                                r |= (uint32_t)c << (8 * b);
                            }
                            w[i] = r;
                        }
                    }
                }
            }
            if (!fast) {
#pragma unroll
                for (int i = 0; i < 16; ++i) {
                    const int64_t p = p0 + i;
                    if (p < begin + j1) {
                        while (p >= E.end) load_entry(a, E.e + 1, E);
                        const Src s = locate(a, E, p - E.begin);
                        uint8_t c = s.c;
                        if (s.field >= 0) {
                            const int64_t src = E.start(s.field) + s.idx;
                            const uint8_t raw = (src >= 0 && (uint64_t)src < a.base_bytes[s.field]) ? a.base[s.field][src] : 0;
                            c = s_lut[s.field][raw];
                            if (CHECK && s.field == 1 && a.lut[1] && c == 0) report_bad(a.status, (E.e << 32) | s.idx);
                        }
                        w[i >> 2] |= (uint32_t)c << (8 * (i & 3));
                    }
                }
            }
            if (!CHECK) {
                uint8_t *dst = a.out + j0;
                if (j1 - j0 == 16) {
                    *reinterpret_cast<uint4 *>(dst) = make_uint4(w[0], w[1], w[2], w[3]);
                } else {
#pragma unroll
                    for (int i = 0; i < 16; ++i)
                        if (i < j1 - j0) dst[i] = (uint8_t)(w[i >> 2] >> (8 * (i & 3)));
                }
            }
        }
    }
}

int fill_args(FmtArgs &a, int format, int line_width, size_t n_entries, const bnpk_field *fields) {
    if (format != BNPK_FMT_FASTQ && format != BNPK_FMT_FASTA && format != BNPK_FMT_FASTA_WRAPPED)
        return set_err(BNPK_E_BADARG, "unknown record format");
    if (format == BNPK_FMT_FASTA_WRAPPED && line_width < 1)
        return set_err(BNPK_E_BADARG, "wrapped FASTA needs line_width >= 1");
    if (!fields) return set_err(BNPK_E_BADARG, "fields must point to three bnpk_field");
    const int n_fields = format == BNPK_FMT_FASTQ ? 3 : 2;
    memset(&a, 0, sizeof(a));
    for (int f = 0; f < n_fields; ++f) {
        if (n_entries && (!fields[f].starts || !fields[f].lens))
            return set_err(BNPK_E_BADARG, f == 2 ? "FASTQ needs a quality field" : "name and sequence fields are required");
        a.base[f] = fields[f].base;
        a.base_bytes[f] = fields[f].base_bytes;
        a.starts[f] = fields[f].starts;
        a.lens[f] = fields[f].lens;
        a.lut[f] = fields[f].lut256;
    }
    a.fmt = format;
    a.width = format == BNPK_FMT_FASTA_WRAPPED ? line_width : 1;
    a.n = (int64_t)n_entries;
    return 0;
}

unsigned fmt_grid(int64_t span_bytes) {
    return grid_cap((size_t)((span_bytes + kFmtTile - 1) / kFmtTile), 8);
}

// --------------------------------------------------------------------------------------------------------------------
// delimited lines (K14)
// --------------------------------------------------------------------------------------------------------------------
constexpr int kDelimThreads = 256;
constexpr int64_t kDelimWindow = 16384;         // output bytes a CTA builds in shared memory at a time

struct DelimColumn {
    int kind;
    const uint8_t *data;
    uint64_t base_bytes;
    const int64_t *starts;
    const int32_t *lens;
};

struct DelimArgs {
    DelimColumn col[BNPK_MAX_OUT_COLUMNS];
    int n_cols;
    int64_t n;                      // lines
    const int64_t *offs;            // int64[n + 1]
    int64_t out_begin, out_end;
    uint8_t *out;
    int64_t *status;
};

// |v| and the number of characters of v in decimal ('-' included); INT64_MIN's magnitude is 2^63
__device__ __forceinline__ int int_width(int64_t v, uint64_t &mag) {
    mag = v < 0 ? 0ull - (uint64_t)v : (uint64_t)v;
    int d = 1;
    uint64_t p = 10;
#pragma unroll
    for (int k = 1; k < 20; ++k, p *= 10) d += mag >= p;
    return d + (v < 0);
}

__device__ __forceinline__ int64_t field_width(const DelimColumn &c, int64_t e) {
    if (c.kind == BNPK_COL_TEXT) return (int64_t)max(c.lens[e], 0);
    if (c.kind == BNPK_COL_STRAND) return 1;
    uint64_t mag;
    return int_width(((const int64_t *)c.data)[e], mag);
}

// exclusive prefix sum of the line sizes (every column, a tab between two, '\n'); offs[n] = total
__global__ void __launch_bounds__(kScanThreads) delimited_offsets_kernel(const __grid_constant__ DelimArgs a,
                                                                         int64_t *offs, uint64_t *ws) {
    exclusive_offsets(a.n, offs, ws, [&](int64_t e) -> uint64_t {
        int64_t size = a.n_cols;
        for (int k = 0; k < a.n_cols; ++k) {
            const DelimColumn &c = a.col[k];
            size += field_width(c, e);
            if (c.kind == BNPK_COL_STRAND && c.data[e] > 2)
                atomicMin((long long *)&a.status[BNPK_ST_BAD_BASE], (long long)(e << 8 | k << 3 | BNPK_BAD_STRAND));
        }
        return (uint64_t)size;
    });
}

// The digits of mag < 10^9 that end at window index `last` (inclusive), `n_digits` of them (leading zeros when the
// part is not the top one); only the indices in [0, kDelimWindow) are written.
__device__ __forceinline__ void put_digits(uint8_t *win, int64_t last, uint32_t part, int n_digits) {
    for (int i = 0; i < n_digits; ++i) {
        const int64_t q = last - i;
        const uint32_t next = part / 10;
        if (q >= 0 && q < kDelimWindow) win[q] = (uint8_t)('0' + (part - next * 10));
        part = next;
    }
}

// A CTA owns the output window [w0, w0 + kDelimWindow) (out-relative, aligned so that out + w0 is 16-byte aligned) and
// builds, one line per thread, the bytes of every line that overlaps it into shared memory; a line that straddles two
// windows is built by both CTAs, each keeping its own bytes.  The window is then stored with 16-byte stores.
__global__ void __launch_bounds__(kDelimThreads) delimited_text_kernel(const __grid_constant__ DelimArgs a) {
    __shared__ __align__(16) uint8_t win[kDelimWindow];
    const int64_t begin = a.out_begin, span = a.out_end - a.out_begin;
    const int mis = (int)(reinterpret_cast<uintptr_t>(a.out) & 15);
    const int64_t n_windows = (span + mis + kDelimWindow - 1) / kDelimWindow;
    for (int64_t w = blockIdx.x; w < n_windows; w += gridDim.x) {
        const int64_t w0 = w * kDelimWindow - mis;                          // out-relative index of win[0]
        const int64_t lo_j = max(w0, (int64_t)0), hi_j = min(w0 + kDelimWindow, span);
        const int64_t lo = find_entry(a.offs, 0, a.n - 1, begin + lo_j);
        const int64_t hi = find_entry(a.offs, lo, a.n - 1, begin + hi_j - 1);
        for (int64_t e = lo + threadIdx.x; e <= hi; e += kDelimThreads) {
            int64_t q = a.offs[e] - begin - w0;                             // window index of the line's next byte
            for (int k = 0; k < a.n_cols; ++k) {
                const DelimColumn &c = a.col[k];
                if (k) {
                    if (q >= 0 && q < kDelimWindow) win[q] = '\t';
                    ++q;
                }
                if (c.kind == BNPK_COL_TEXT) {
                    const int64_t len = max(c.lens[e], 0);
                    const int64_t src = len ? c.starts[e] : 0;
                    for (int64_t i = max(-q, (int64_t)0), i1 = min(len, kDelimWindow - q); i < i1; ++i) {
                        const int64_t b = src + i;
                        win[q + i] = b >= 0 && (uint64_t)b < c.base_bytes ? c.data[b] : 0;
                    }
                    q += len;
                } else if (c.kind == BNPK_COL_STRAND) {
                    const uint8_t code = c.data[e];
                    if (q >= 0 && q < kDelimWindow) win[q] = code == 0 ? '+' : code == 1 ? '-' : '.';
                    ++q;
                } else {
                    const int64_t v = ((const int64_t *)c.data)[e];
                    uint64_t mag;
                    const int width = int_width(v, mag);
                    if (q + width > 0 && q < kDelimWindow) {
                        if (v < 0 && q >= 0) win[q] = '-';
                        // split once at 10^9 and 10^18, then every digit comes from 32-bit arithmetic
                        const uint64_t top = mag / 1000000000ull;
                        const uint32_t low = (uint32_t)(mag - top * 1000000000ull);
                        const uint32_t mid = (uint32_t)(top % 1000000000ull), high = (uint32_t)(top / 1000000000ull);
                        const int n_digits = width - (v < 0);
                        const int64_t last = q + width - 1;
                        put_digits(win, last, low, min(n_digits, 9));
                        if (n_digits > 9) put_digits(win, last - 9, mid, min(n_digits - 9, 9));
                        if (n_digits > 18) put_digits(win, last - 18, high, n_digits - 18);
                    }
                    q += width;
                }
            }
            if (q >= 0 && q < kDelimWindow) win[q] = '\n';
        }
        __syncthreads();
        for (int64_t u = threadIdx.x; u < kDelimWindow / 16; u += kDelimThreads) {
            const int64_t j0 = w0 + 16 * u;
            if (j0 + 16 <= lo_j || j0 >= hi_j) continue;
            if (j0 >= lo_j && j0 + 16 <= hi_j) {
                *reinterpret_cast<uint4 *>(a.out + j0) = *reinterpret_cast<const uint4 *>(win + 16 * u);
            } else {
                for (int i = 0; i < 16; ++i)
                    if (j0 + i >= lo_j && j0 + i < hi_j) a.out[j0 + i] = win[16 * u + i];
            }
        }
        __syncthreads();                                                    // the window is free again
    }
}

int fill_delim(DelimArgs &a, const bnpk_out_column *columns, int n_columns, size_t n_lines) {
    if (!columns || n_columns < 1 || n_columns > BNPK_MAX_OUT_COLUMNS)
        return set_err(BNPK_E_BADARG, "1 to BNPK_MAX_OUT_COLUMNS columns are required");
    memset(&a, 0, sizeof(a));
    for (int k = 0; k < n_columns; ++k) {
        const bnpk_out_column &c = columns[k];
        if (c.kind != BNPK_COL_TEXT && c.kind != BNPK_COL_INT && c.kind != BNPK_COL_STRAND)
            return set_err(BNPK_E_BADARG, "a written column is BNPK_COL_TEXT, BNPK_COL_INT or BNPK_COL_STRAND");
        if (n_lines && (!c.data || (c.kind == BNPK_COL_TEXT && (!c.starts || !c.lens))))
            return set_err(BNPK_E_BADARG, "a column misses its data, starts or lens");
        a.col[k] = DelimColumn{c.kind, (const uint8_t *)c.data, (uint64_t)c.base_bytes, c.starts, c.lens};
    }
    a.n_cols = n_columns;
    a.n = (int64_t)n_lines;
    return 0;
}

}  // namespace
}  // namespace bnpk

using namespace bnpk;

extern "C" {

int bnpk_format_offsets(int format, int line_width, size_t n_entries, const bnpk_field *fields, int64_t *out_offsets,
                        int64_t *status, void *workspace, size_t workspace_bytes, void *stream) {
    FmtArgs a;
    if (int rc = fill_args(a, format, line_width, n_entries, fields)) return rc;
    cudaStream_t st = (cudaStream_t)stream;
    if (n_entries == 0) {
        BNPK_CUDA(cudaMemsetAsync(out_offsets, 0, sizeof(int64_t), st));
        return 0;
    }
    size_t n_tiles;
    if (int rc = scan_workspace(n_entries, 1, workspace, workspace_bytes, st, n_tiles)) return rc;
    if (int rc = launch("format_offsets_kernel", format_offsets_kernel, grid_cap(n_tiles, 4), kScanThreads, 0, st, false,
                        a, out_offsets, (uint64_t *)workspace))
        return rc;
    if (!a.lut[1]) return 0;                 // raw text: every byte is written as it is
    if (!status) return set_err(BNPK_E_BADARG, "a sequence LUT needs a status block for the bad-base report");
    a.offs = out_offsets;
    a.status = status;
    // the total is on the device: a grid for the average case, every CTA loops over tiles up to offs[n]
    return launch("format_kernel<check>", format_kernel<true>, (unsigned)sm_count() * 8, kFmtThreads, 0, st, false, a);
}

int bnpk_format_records(int format, int line_width, size_t n_entries, const bnpk_field *fields,
                        const int64_t *out_offsets, int64_t out_begin, int64_t out_end, uint8_t *out, void *stream) {
    FmtArgs a;
    if (int rc = fill_args(a, format, line_width, n_entries, fields)) return rc;
    if (out_end < out_begin || out_begin < 0) return set_err(BNPK_E_BADARG, "need 0 <= out_begin <= out_end");
    if (out_end == out_begin) return 0;
    if (!out) return set_err(BNPK_E_BADARG, "out is NULL for a non-empty range");
    if (n_entries == 0 || !out_offsets) return set_err(BNPK_E_BADARG, "a non-empty range needs entries and their offsets");
    a.offs = out_offsets;
    a.out_begin = out_begin;
    a.out_end = out_end;
    a.out = out;
    return launch("format_kernel", format_kernel<false>, fmt_grid(out_end - out_begin), kFmtThreads, 0,
                  (cudaStream_t)stream, false, a);
}

int bnpk_delimited_offsets(const bnpk_out_column *columns, int n_columns, size_t n_lines, int64_t *out_offsets,
                           int64_t *status, void *workspace, size_t workspace_bytes, void *stream) {
    DelimArgs a;
    if (int rc = fill_delim(a, columns, n_columns, n_lines)) return rc;
    if (!out_offsets) return set_err(BNPK_E_BADARG, "out_offsets is required");
    cudaStream_t st = (cudaStream_t)stream;
    if (n_lines == 0) {
        BNPK_CUDA(cudaMemsetAsync(out_offsets, 0, sizeof(int64_t), st));
        return 0;
    }
    if (!status || !workspace) return set_err(BNPK_E_BADARG, "status and workspace are required");
    a.status = status;
    size_t n_tiles;
    if (int rc = scan_workspace(n_lines, 1, workspace, workspace_bytes, st, n_tiles)) return rc;
    return launch("delimited_offsets_kernel", delimited_offsets_kernel, grid_cap(n_tiles, 4), kScanThreads, 0, st,
                  false, a, out_offsets, (uint64_t *)workspace);
}

int bnpk_delimited_format(const bnpk_out_column *columns, int n_columns, size_t n_lines, const int64_t *out_offsets,
                          int64_t out_begin, int64_t out_end, uint8_t *out, void *stream) {
    DelimArgs a;
    if (int rc = fill_delim(a, columns, n_columns, n_lines)) return rc;
    if (out_end < out_begin || out_begin < 0) return set_err(BNPK_E_BADARG, "need 0 <= out_begin <= out_end");
    if (out_end == out_begin) return 0;
    if (!out) return set_err(BNPK_E_BADARG, "out is NULL for a non-empty range");
    if (n_lines == 0 || !out_offsets) return set_err(BNPK_E_BADARG, "a non-empty range needs lines and their offsets");
    a.offs = out_offsets;
    a.out_begin = out_begin;
    a.out_end = out_end;
    a.out = out;
    const int64_t windows = (out_end - out_begin + 15 + kDelimWindow - 1) / kDelimWindow;
    return launch("delimited_text_kernel", delimited_text_kernel, grid_cap((size_t)windows, 8), kDelimThreads, 0,
                  (cudaStream_t)stream, false, a);
}

}  // extern "C"
