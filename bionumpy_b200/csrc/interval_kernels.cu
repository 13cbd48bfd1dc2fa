// interval_kernels.cu -- BED columns, contig names and interval sequences on the device
// (DelimitedBuffer.from_raw_buffer / _get_field_by_number io/delimited_buffers.py:52-316, IndexedFasta.get_interval_sequences
// io/indexed_fasta.py:165-206, get_sequences / get_strand_specific_sequences sequence/dna.py:68-106).
//
// delimited_columns_kernel: a CTA takes 128 consecutive lines, stages the bytes they span into shared memory with
//   aligned 16-byte loads (lines of 20-100 bytes: 2.5-12.5 KiB), and each thread then walks one line out of shared
//   memory, column by column.  A span that does not fit is read from global memory instead.
// name_lookup_kernel: one thread per row, a binary search of the sorted name table with a full byte compare.
// interval_check_kernel: one thread per row; validates the interval and writes its length.
// interval_copy_kernel: eight lanes per row; every 16-byte output unit (aligned on the output address) whose source
//   lies on one line of the file is one unaligned 16-byte gather and one vector store, reversed and complemented in
//   registers for a '-' row; the units at the row's ends and those that straddle a line end go byte by byte.
// attribute_values_kernel: one warp per row of a GTF/GFF attribute column, 32-byte windows balloted into masks of
//   ';', '"', ' ' and '=' and walked one attribute boundary at a time (GTFEntry._get_attributes, datatypes/gtf.py).
#include "bnpk_host.h"

namespace bnpk {

namespace {

constexpr int kColThreads = 128;
constexpr int kColStage = 16384;
constexpr int kCopyThreads = 256;
constexpr int kLanesPerRow = 8;
constexpr int64_t kFlatLine = (int64_t)1 << 62;   // the flat mode's "line": no line end is ever reached

struct ColArgs {
    const uint8_t *chunk;
    const int64_t *starts;
    const int32_t *lens;
    int64_t n_lines;
    int n_columns;
    int kind[BNPK_MAX_COLUMNS];
    void *out[BNPK_MAX_COLUMNS];
    int32_t *out_lens[BNPK_MAX_COLUMNS];
    int64_t *status;
};

__global__ void __launch_bounds__(kColThreads) delimited_columns_kernel(const __grid_constant__ ColArgs a) {
    __shared__ uint4 s_stage[kColStage / 16];
    __shared__ int s_kind[BNPK_MAX_COLUMNS];
    __shared__ void *s_out[BNPK_MAX_COLUMNS];
    __shared__ int32_t *s_lens[BNPK_MAX_COLUMNS];
    __shared__ int s_first_tabs, s_cr;
    const int tid = threadIdx.x;
    if (tid < BNPK_MAX_COLUMNS) {
        s_kind[tid] = tid < a.n_columns ? a.kind[tid] : BNPK_COL_SKIP;
        s_out[tid] = a.out[tid];
        s_lens[tid] = a.out_lens[tid];
    }
    if (tid < 32) {
        // the first line's tab count and whether it ends in '\r' (DelimitedBuffer._get_n_fields,
        // _modify_for_carriage_return)
        const int64_t s0 = a.starts[0];
        const int32_t l0 = a.lens[0];
        int tabs = 0;
        for (int64_t i = tid; i < l0; i += 32) tabs += a.chunk[s0 + i] == '\t';
#pragma unroll
        for (int o = 16; o; o >>= 1) tabs += __shfl_xor_sync(0xffffffffu, tabs, o);
        if (tid == 0) {
            s_first_tabs = tabs;
            s_cr = l0 > 0 && a.chunk[s0 + l0 - 1] == '\r';
        }
    }
    __syncthreads();
    const int first_tabs = s_first_tabs;
    const bool cr = s_cr;
    const uint8_t *s_bytes = reinterpret_cast<const uint8_t *>(s_stage);
    for (int64_t l0 = (int64_t)blockIdx.x * kColThreads; l0 < a.n_lines; l0 += (int64_t)gridDim.x * kColThreads) {
        const int64_t l1 = min(l0 + kColThreads, a.n_lines);
        const uintptr_t lo = reinterpret_cast<uintptr_t>(a.chunk + a.starts[l0]) & ~(uintptr_t)15;
        const uintptr_t hi = reinterpret_cast<uintptr_t>(a.chunk + a.starts[l1 - 1] + a.lens[l1 - 1]);
        const bool staged = hi - lo <= (uintptr_t)kColStage;
        __syncthreads();    // the previous lines are done with the stage
        if (staged) {
            const uint4 *src = reinterpret_cast<const uint4 *>(lo);
            const int n_units = (int)((hi - lo + 15) / 16);
            for (int u = tid; u < n_units; u += kColThreads) s_stage[u] = ld_stream(src + u);
        }
        __syncthreads();
        const int64_t line = l0 + tid;
        if (line >= l1) continue;
        const int64_t s = a.starts[line];
        int32_t L = a.lens[line];
        const uint8_t *g = a.chunk + s;
        const uint8_t *p = staged ? s_bytes + (reinterpret_cast<uintptr_t>(g) - lo) : g;
        if (cr && L > 0 && p[L - 1] == '\r') --L;
        int col = 0;
        int32_t f0 = 0;           // first byte of the current field
        int64_t val = 0;
        int nd = 0;               // digits of the current field
        bool neg = false, bad = false;
        int64_t fault = INT64_MAX;
        for (int32_t i = 0; i <= L; ++i) {
            const uint8_t c = i < L ? p[i] : (uint8_t)'\t';
            const int kind = col < BNPK_MAX_COLUMNS ? s_kind[col] : BNPK_COL_SKIP;
            if (c != '\t') {
                if (kind == BNPK_COL_INT || kind == BNPK_COL_INT_OR_DOT) {
                    const unsigned d = (unsigned)c - '0';
                    if (d < 10) {
                        val = val * 10 + d;
                        ++nd;
                    } else if (i == f0 && (c == '-' || c == '+')) {
                        neg = c == '-';
                    } else {
                        bad = true;
                    }
                }
                continue;
            }
            const int32_t flen = i - f0;
            if (kind == BNPK_COL_TEXT) {
                reinterpret_cast<int64_t *>(s_out[col])[line] = s + f0;
                s_lens[col][line] = flen;
            } else if (kind == BNPK_COL_INT || kind == BNPK_COL_INT_OR_DOT) {
                const bool dot = kind == BNPK_COL_INT_OR_DOT && flen == 1 && p[f0] == '.';
                if (!dot && (bad || nd == 0 || nd > 18)) fault = min(fault, fault_column(line, min(col, 31), BNPK_BAD_INT));
                reinterpret_cast<int64_t *>(s_out[col])[line] = dot ? 0 : neg ? -val : val;
            } else if (kind == BNPK_COL_STRAND) {
                const uint8_t b = flen == 1 ? p[f0] : 0;
                const int code = b == '+' ? 0 : b == '-' ? 1 : b == '.' ? 2 : -1;
                if (code < 0) fault = min(fault, fault_column(line, min(col, 31), BNPK_BAD_STRAND));
                reinterpret_cast<uint8_t *>(s_out[col])[line] = (uint8_t)max(code, 0);
            }
            ++col;
            f0 = i + 1;
            val = 0;
            nd = 0;
            neg = bad = false;
        }
        // a line with another tab count is reported as that, before whatever its fields held
        if (col - 1 != first_tabs) fault = fault_column(line, min(col, 31), BNPK_BAD_TABS);
        else if (col < a.n_columns) fault = fault_column(line, min(col, 31), BNPK_BAD_COLUMNS);
        if (fault != INT64_MAX) report_fault(a.status, fault);
    }
}

// < 0, 0, > 0 as row bytes r[0..rl) compare with name bytes q[0..ql): bytewise, then the shorter first
__device__ __forceinline__ int name_cmp(const uint8_t *r, int64_t rl, const uint8_t *q, int64_t ql) {
    const int64_t m = min(rl, ql);
    for (int64_t i = 0; i < m; ++i) {
        const int d = (int)r[i] - (int)q[i];
        if (d) return d;
    }
    return rl < ql ? -1 : rl > ql ? 1 : 0;
}

__global__ void __launch_bounds__(256) name_lookup_kernel(const uint8_t *base, size_t base_bytes, const int64_t *starts,
                                                          const int32_t *lens, size_t n_rows, const uint8_t *names,
                                                          const int64_t *name_offsets, int64_t n_names, int32_t *out_ids,
                                                          int64_t *status) {
    for (size_t r = (size_t)blockIdx.x * blockDim.x + threadIdx.x; r < n_rows; r += (size_t)gridDim.x * blockDim.x) {
        const int64_t s = starts[r], l = max(lens[r], 0);
        int32_t id = -1;
        if (s >= 0 && (uint64_t)(s + l) <= base_bytes) {
            int64_t lo = 0, hi = n_names - 1;
            while (lo <= hi) {
                const int64_t mid = (lo + hi) >> 1;
                const int64_t q0 = name_offsets[mid];
                const int c = name_cmp(base + s, l, names + q0, name_offsets[mid + 1] - q0);
                if (c == 0) {
                    id = (int32_t)mid;
                    break;
                }
                if (c < 0) hi = mid - 1;
                else lo = mid + 1;
            }
        }
        out_ids[r] = id;
        if (id < 0) report_fault(status, (int64_t)r);
    }
}

struct Contig {
    int64_t offset, lenc, lenb, len;
};

struct GatherArgs {
    const uint8_t *file;
    uint64_t file_bytes;
    int64_t n_rows;
    const int32_t *ids;
    const int64_t *c_offset;
    const int32_t *c_lenc, *c_lenb;
    const int64_t *c_len;
    int64_t n_contigs;
    const int64_t *start, *stop;
    const uint8_t *strand;
    const uint8_t *comp;
    int32_t *row_lens;
    const int64_t *offs;
    uint8_t *out;
    int64_t *status;
};

// the contig of row r; false for a contig id outside the table
__device__ __forceinline__ bool contig_of(const GatherArgs &a, int64_t r, Contig &c) {
    if (!a.ids) {
        c = Contig{0, kFlatLine, kFlatLine, (int64_t)a.file_bytes};
        return true;
    }
    const int32_t id = a.ids[r];
    if (id < 0 || id >= a.n_contigs) return false;
    c = Contig{a.c_offset[id], max(a.c_lenc[id], 1), max(a.c_lenb[id], 1), a.c_len[id]};
    return true;
}

// file byte of base p of the contig
__device__ __forceinline__ int64_t file_pos(const Contig &c, int64_t p) {
    const int64_t line = p / c.lenc;
    return c.offset + line * c.lenb + (p - line * c.lenc);
}

__global__ void __launch_bounds__(256) interval_check_kernel(const __grid_constant__ GatherArgs a) {
    for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < a.n_rows; r += (int64_t)gridDim.x * blockDim.x) {
        const int64_t s = a.start[r], e = a.stop[r];
        Contig c;
        bool ok = contig_of(a, r, c) && s >= 0 && e >= s && e <= c.len && e - s <= INT32_MAX;
        if (ok && e > s) ok = c.offset >= 0 && (uint64_t)file_pos(c, e - 1) < a.file_bytes;
        a.row_lens[r] = ok ? (int32_t)(e - s) : 0;
        if (!ok) report_fault(a.status, r);
    }
}

__global__ void __launch_bounds__(kCopyThreads) interval_copy_kernel(const __grid_constant__ GatherArgs a) {
    __shared__ uint8_t s_comp[256];
    for (int i = threadIdx.x; i < 256; i += kCopyThreads) s_comp[i] = a.comp ? a.comp[i] : (uint8_t)i;
    __syncthreads();
    const int sub = threadIdx.x % kLanesPerRow;
    const int64_t group = ((int64_t)blockIdx.x * kCopyThreads + threadIdx.x) / kLanesPerRow;
    const int64_t n_groups = (int64_t)gridDim.x * kCopyThreads / kLanesPerRow;
    for (int64_t r = group; r < a.n_rows; r += n_groups) {
        const int64_t o = a.offs[r], L = a.offs[r + 1] - o;
        Contig c;
        if (L <= 0 || !contig_of(a, r, c)) continue;
        const int64_t s = a.start[r];
        const bool rev = a.strand && a.strand[r];
        uint8_t *dst = a.out + o;
        // out-relative units: a head of `head` bytes up to the first 16-byte aligned output address, then whole units
        const int64_t head = min((int64_t)((16 - (reinterpret_cast<uintptr_t>(dst) & 15)) & 15), L);
        const int64_t n_units = (head ? 1 : 0) + (L - head + 15) / 16;
        for (int64_t u = sub; u < n_units; u += kLanesPerRow) {
            const int64_t j0 = head ? (u == 0 ? 0 : head + (u - 1) * 16) : u * 16;
            const int64_t j1 = min(head && u == 0 ? head : j0 + 16, L);
            // source bases of the unit: [b0, b0 + 16), forwards or backwards
            const int64_t b0 = rev ? s + L - j0 - 16 : s + j0;
            if (j1 - j0 == 16 && b0 / c.lenc == (b0 + 15) / c.lenc) {
                uint32_t w[4];
                load16(a.file + file_pos(c, b0), w);
                if (rev) {
                    uint32_t t[4];
#pragma unroll
                    for (int i = 0; i < 4; ++i) {
                        const uint32_t x = w[3 - i];
                        t[i] = (uint32_t)s_comp[x >> 24] | (uint32_t)s_comp[(x >> 16) & 255] << 8 |
                               (uint32_t)s_comp[(x >> 8) & 255] << 16 | (uint32_t)s_comp[x & 255] << 24;
                    }
                    *reinterpret_cast<uint4 *>(dst + j0) = make_uint4(t[0], t[1], t[2], t[3]);
                } else {
                    *reinterpret_cast<uint4 *>(dst + j0) = make_uint4(w[0], w[1], w[2], w[3]);
                }
            } else {
                for (int64_t j = j0; j < j1; ++j) {
                    const uint8_t v = a.file[file_pos(c, rev ? s + L - 1 - j : s + j)];
                    dst[j] = rev ? s_comp[v] : v;
                }
            }
        }
    }
}

// attribute_values_kernel: one warp per row of a GTF/GFF attribute column.  The warp reads the row in 32-byte windows,
// one byte per lane, and ballots the window's ';', '"', ' ' and '=' into four masks.  Every lane then runs the same
// scalar walk over those masks: each step takes the first bit of the mask its state waits for, so the walk costs one
// step per attribute boundary, not per byte, and the bytes are read once, coalesced.  At a key's end the lanes compare
// the key with the requested keys of its length (one byte per lane).  Lane k keeps key k's value.
constexpr int kAttrThreads = 256;
enum AttrState { kPre, kKey, kGap, kQuote, kTail, kVal };

// the bits of a window starting at w that lie at or after position cur
__device__ __forceinline__ unsigned from_mask(int32_t cur, int32_t w) {
    return cur <= w ? ~0u : cur - w >= 32 ? 0u : ~0u << (cur - w);
}

struct AttrArgs {
    const uint8_t *base;
    uint64_t base_bytes;
    const int64_t *starts;
    const int32_t *lens;
    int64_t n_rows;
    const uint8_t *select;
    int n_keys;
    int gff;
    int key_len[BNPK_MAX_KEYS];
    uint8_t keys[BNPK_MAX_KEYS][BNPK_MAX_KEY_LEN];
    int64_t *out_starts;
    int32_t *out_lens;
    int64_t *status;
};

__global__ void __launch_bounds__(kAttrThreads) attribute_values_kernel(const __grid_constant__ AttrArgs a) {
    __shared__ uint8_t s_keys[BNPK_MAX_KEYS][BNPK_MAX_KEY_LEN];
    for (int i = threadIdx.x; i < BNPK_MAX_KEYS * BNPK_MAX_KEY_LEN; i += kAttrThreads)
        s_keys[i / BNPK_MAX_KEY_LEN][i % BNPK_MAX_KEY_LEN] = a.keys[i / BNPK_MAX_KEY_LEN][i % BNPK_MAX_KEY_LEN];
    __syncthreads();
    const int lane = threadIdx.x & 31;
    const unsigned all = (1u << a.n_keys) - 1;
    const int64_t n_warps = (int64_t)gridDim.x * (kAttrThreads / 32);
    for (int64_t r = ((int64_t)blockIdx.x * kAttrThreads + threadIdx.x) / 32; r < a.n_rows; r += n_warps) {
        const int64_t s = a.starts[r];
        int64_t my_start = s;
        int32_t my_len = 0;
        if (a.select && !a.select[r]) {
            if (lane < a.n_keys) {
                a.out_starts[lane * a.n_rows + r] = my_start;
                a.out_lens[lane * a.n_rows + r] = my_len;
            }
            continue;
        }
        int32_t L = max(a.lens[r], 0);
        if (s < 0 || (uint64_t)s + (uint64_t)L > a.base_bytes) L = 0;
        const uint8_t *row = a.base + (s < 0 ? 0 : s);
        int state = kPre;
        int32_t cur = 0, ks = 0, vs = 0, last_ns = -1;
        unsigned found = 0, match = 0;
        // record the value [v0, v0 + n) of the keys in `match` that have none yet
        auto record = [&](int32_t v0, int32_t n) {
            const unsigned fresh = match & ~found;
            found |= fresh;
            if (fresh >> lane & 1) {
                my_start = s + v0;
                my_len = n;
            }
        };
        for (int32_t w = 0; w < L && found != all; w += 32) {
            const int32_t i = w + lane;
            const uint8_t c = i < L ? row[i] : (uint8_t)0;
            const unsigned valid = L - w >= 32 ? ~0u : (1u << (L - w)) - 1;
            const unsigned semi = __ballot_sync(~0u, c == ';');
            const unsigned quote = __ballot_sync(~0u, c == '"');
            const unsigned nonsp = ~__ballot_sync(~0u, c == ' ') & valid;
            const unsigned key_end = a.gff ? (__ballot_sync(~0u, c == '=') | semi) : (~nonsp & valid) | semi;
            for (;;) {
                const unsigned from = from_mask(cur, w);
                const unsigned wait = state == kPre || state == kGap ? nonsp
                                      : state == kKey              ? key_end
                                      : state == kQuote            ? quote
                                                                   : semi;
                const unsigned ev = wait & from;
                if (!ev) break;
                const int bit = __ffs(ev) - 1;
                const int32_t p = w + bit;
                const bool at_semi = semi >> bit & 1;
                cur = p + 1;
                if (state == kPre) {
                    if (!at_semi) {
                        ks = p;
                        cur = p;
                        state = kKey;
                    }
                } else if (state == kKey) {
                    match = 0;
                    if (at_semi) {
                        state = kPre;       // an attribute without a value
                        continue;
                    }
                    const int32_t n = p - ks;
                    unsigned cand = 0;
#pragma unroll
                    for (int k = 0; k < BNPK_MAX_KEYS; ++k)
                        if (a.key_len[k] == n && !(found >> k & 1)) cand |= 1u << k;
                    cand &= all;
                    if (cand) {
                        const uint8_t b = lane < n ? row[ks + lane] : (uint8_t)0;
                        while (cand) {
                            const int k = __ffs(cand) - 1;
                            cand &= cand - 1;
                            if (__ballot_sync(~0u, lane >= n || b == s_keys[k][lane]) == ~0u) match |= 1u << k;
                        }
                    }
                    if (a.gff) {
                        vs = p + 1;
                        state = kVal;
                    } else {
                        state = kGap;
                    }
                } else if (state == kGap) {
                    if (at_semi) {
                        record(p, 0);
                        state = kPre;
                    } else if (quote >> bit & 1) {
                        vs = p + 1;
                        state = kQuote;
                    } else {
                        vs = last_ns = p;
                        state = kVal;
                    }
                } else if (state == kQuote) {
                    record(vs, p - vs);
                    state = kTail;
                } else if (state == kTail) {
                    state = kPre;
                } else {
                    if (a.gff) {
                        record(vs, p - vs);
                    } else {
                        const unsigned before = nonsp & from & ((1u << bit) - 1);
                        const int32_t last = before ? w + 31 - __clz(before) : last_ns;
                        record(vs, last + 1 - vs);
                    }
                    state = kPre;
                }
            }
            if (state == kVal && !a.gff) {
                const unsigned ns = nonsp & from_mask(cur, w);
                if (ns) last_ns = w + 31 - __clz(ns);
            }
        }
        if (found != all) {
            if (state == kGap) record(L, 0);
            else if (state == kQuote) record(vs, L - vs);
            else if (state == kVal) record(vs, (a.gff ? L : last_ns + 1) - vs);
        }
        if (lane < a.n_keys) {
            a.out_starts[lane * a.n_rows + r] = my_start;
            a.out_lens[lane * a.n_rows + r] = my_len;
            if (!(found >> lane & 1)) report_fault(a.status, fault_column(r, lane, BNPK_BAD_ATTRIBUTE));
        }
    }
}

}  // namespace
}  // namespace bnpk

using namespace bnpk;

extern "C" {

int bnpk_delimited_columns(const uint8_t *chunk, size_t /* n: the lines lie inside it */, const int64_t *line_starts, const int32_t *line_lens,
                           size_t n_lines, const bnpk_column *columns, int n_columns, int64_t *status, void *stream) {
    if (n_columns < 1 || n_columns > BNPK_MAX_COLUMNS || !columns)
        return set_err(BNPK_E_BADARG, "n_columns must be 1..BNPK_MAX_COLUMNS with a host array of bnpk_column");
    ColArgs a;
    memset(&a, 0, sizeof(a));
    for (int c = 0; c < n_columns; ++c) {
        const int k = columns[c].kind;
        if (k < BNPK_COL_SKIP || k > BNPK_COL_STRAND) return set_err(BNPK_E_BADARG, "unknown column kind");
        if (k != BNPK_COL_SKIP && !columns[c].out) return set_err(BNPK_E_BADARG, "a named column needs its output");
        if (k == BNPK_COL_TEXT && !columns[c].lens) return set_err(BNPK_E_BADARG, "a text column needs its lens output");
        a.kind[c] = k;
        a.out[c] = columns[c].out;
        a.out_lens[c] = columns[c].lens;
    }
    if (n_lines == 0) return 0;
    if (!chunk || !line_starts || !line_lens || !status)
        return set_err(BNPK_E_BADARG, "chunk, line_starts, line_lens and status are required");
    a.chunk = chunk;
    a.starts = line_starts;
    a.lens = line_lens;
    a.n_lines = (int64_t)n_lines;
    a.n_columns = n_columns;
    a.status = status;
    return launch("delimited_columns_kernel", delimited_columns_kernel,
                  grid_cap((n_lines + kColThreads - 1) / kColThreads, 16), kColThreads, 0, (cudaStream_t)stream, false, a);
}

int bnpk_name_lookup(const uint8_t *base, size_t base_bytes, const int64_t *starts, const int32_t *lens, size_t n_rows,
                     const uint8_t *names, const int64_t *name_offsets, size_t n_names, int32_t *out_ids,
                     int64_t *status, void *stream) {
    if (n_rows == 0) return 0;
    if (!base || !starts || !lens || !name_offsets || !out_ids || !status || (n_names && !names))
        return set_err(BNPK_E_BADARG, "base, starts, lens, names, name_offsets, out_ids and status are required");
    return launch("name_lookup_kernel", name_lookup_kernel, grid_cap((n_rows + 255) / 256, 8), 256, 0,
                  (cudaStream_t)stream, false, base, base_bytes, starts, lens, n_rows, names, name_offsets,
                  (int64_t)n_names, out_ids, status);
}

int bnpk_interval_gather(const uint8_t *file, size_t file_bytes, size_t n_rows, const int32_t *ids,
                         const int64_t *contig_offset, const int32_t *lenc, const int32_t *lenb, const int64_t *contig_len,
                         size_t n_contigs, const int64_t *start, const int64_t *stop, const uint8_t *strand,
                         const uint8_t *complement_lut256, int32_t *row_lens, const int64_t *out_offsets, uint8_t *out,
                         int64_t *status, void *stream) {
    if (ids && (!contig_offset || !lenc || !lenb || !contig_len))
        return set_err(BNPK_E_BADARG, "contig ids need the contig table (offset, lenc, lenb, length)");
    if (strand && !complement_lut256) return set_err(BNPK_E_BADARG, "a strand flag needs complement_lut256");
    if (n_rows == 0) return 0;
    if (!file || !start || !stop) return set_err(BNPK_E_BADARG, "file, start and stop are required");
    GatherArgs a{file, (uint64_t)file_bytes, (int64_t)n_rows, ids, contig_offset, lenc, lenb, contig_len,
                 (int64_t)n_contigs, start, stop, strand, complement_lut256, row_lens, out_offsets, out, status};
    if (!out) {
        if (!row_lens || !status) return set_err(BNPK_E_BADARG, "the check pass needs row_lens and status");
        return launch("interval_check_kernel", interval_check_kernel, grid_cap((n_rows + 255) / 256, 8), 256, 0,
                      (cudaStream_t)stream, false, a);
    }
    if (!out_offsets) return set_err(BNPK_E_BADARG, "the copy pass needs out_offsets");
    const size_t rows_per_cta = kCopyThreads / kLanesPerRow;
    return launch("interval_copy_kernel", interval_copy_kernel, grid_cap((n_rows + rows_per_cta - 1) / rows_per_cta, 8),
                  kCopyThreads, 0, (cudaStream_t)stream, false, a);
}

int bnpk_attribute_values(const uint8_t *base, size_t base_bytes, const int64_t *starts, const int32_t *lens,
                          size_t n_rows, const uint8_t *select, const uint8_t *keys, const int64_t *key_offsets,
                          int n_keys, int mode, int64_t *out_starts, int32_t *out_lens, int64_t *status, void *stream) {
    if (n_keys < 1 || n_keys > BNPK_MAX_KEYS || !keys || !key_offsets)
        return set_err(BNPK_E_BADARG, "1 to BNPK_MAX_KEYS keys, as a host table (keys, key_offsets)");
    if (mode != BNPK_ATTR_GTF && mode != BNPK_ATTR_GFF) return set_err(BNPK_E_BADARG, "unknown attribute mode");
    AttrArgs a;
    memset(&a, 0, sizeof(a));
    for (int k = 0; k < n_keys; ++k) {
        const int64_t n = key_offsets[k + 1] - key_offsets[k];
        if (n < 1 || n > BNPK_MAX_KEY_LEN) return set_err(BNPK_E_BADARG, "a key holds 1 to BNPK_MAX_KEY_LEN bytes");
        a.key_len[k] = (int)n;
        memcpy(a.keys[k], keys + key_offsets[k], (size_t)n);
    }
    if (n_rows == 0) return 0;
    if (!base || !starts || !lens || !out_starts || !out_lens || !status)
        return set_err(BNPK_E_BADARG, "base, starts, lens, out_starts, out_lens and status are required");
    a.base = base;
    a.base_bytes = (uint64_t)base_bytes;
    a.starts = starts;
    a.lens = lens;
    a.n_rows = (int64_t)n_rows;
    a.select = select;
    a.n_keys = n_keys;
    a.gff = mode == BNPK_ATTR_GFF;
    a.out_starts = out_starts;
    a.out_lens = out_lens;
    a.status = status;
    const size_t rows_per_cta = kAttrThreads / 32;
    return launch("attribute_values_kernel", attribute_values_kernel,
                  grid_cap((n_rows + rows_per_cta - 1) / rows_per_cta, 8), kAttrThreads, 0, (cudaStream_t)stream, false,
                  a);
}

}  // extern "C"
