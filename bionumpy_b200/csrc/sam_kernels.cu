// sam_kernels.cu -- SAM text alignments on the device (SAMBuffer, io/buffers/sam.py; SAMEntry, datatypes/__init__.py).
//
// sam_columns_kernel: one warp per line (DESIGN §3 K16).  Each lane loads one aligned 16-byte unit, so a step of the
//   warp covers 512 bytes; bytes outside the line are masked, the lanes' tab masks are counted with a warp prefix of
//   __popc and the first 11 tab offsets go to shared memory.  The walk stops at the window that holds the 11th tab:
//   the bytes after it are the `extra` view and are never read.  Lanes 0..10 then write one mandatory column each
//   (text as start and length, the five integers parsed from their few bytes) and lane 11 the extra view.
// cigar_count_kernel / cigar_unpack_kernel: one thread per row of CIGAR text.  The count pass validates the row and
//   gives its op count and reference length; the unpack pass writes the ops at the exclusive scan of the counts
//   (bnpk_row_offsets), never more than its row's share of the output.
#include "bnpk_host.h"

namespace bnpk {

namespace {

constexpr int kSamThreads = 256;
constexpr int kSamWarps = kSamThreads / 32;
constexpr int kSamTabs = 11;            // the tab after the 11th column begins `extra`
constexpr int kMaxDigits = 18;          // of an integer column, after an optional sign
constexpr int kMaxCigarDigits = 9;

// column c's output rows: text (start, length) or an integer value; -1 = no such row
__device__ __constant__ const int8_t kColStart[kSamTabs] = {
    BNPK_SAM_F_NAME_START, -1, BNPK_SAM_F_RNAME_START, -1, -1, BNPK_SAM_F_CIGAR_START, BNPK_SAM_F_RNEXT_START, -1, -1,
    BNPK_SAM_F_SEQ_START, BNPK_SAM_F_QUAL_START};
__device__ __constant__ const int8_t kColValue[kSamTabs] = {
    -1, BNPK_SAM_F_FLAG, -1, BNPK_SAM_F_POS, BNPK_SAM_F_MAPQ, -1, -1, BNPK_SAM_F_PNEXT, BNPK_SAM_F_TLEN, -1, -1};

// bit i = "byte i of the unit is '\t'" (exact: a zero byte of w ^ 0x09.. has bit 7 set after the carry-free test)
__device__ __forceinline__ uint32_t tab_msb(uint32_t w) {
    const uint32_t x = w ^ 0x09090909u;
    return ~(((x & 0x7F7F7F7Fu) + 0x7F7F7F7Fu) | x) & 0x80808080u;
}
__device__ __forceinline__ uint32_t tab_mask16(const uint4 q) {
    uint32_t lo = __dp4a(tab_msb(q.x), 0x08040201u, 0u);
    lo = __dp4a(tab_msb(q.y), 0x80402010u, lo);
    uint32_t hi = __dp4a(tab_msb(q.z), 0x08040201u, 0u);
    hi = __dp4a(tab_msb(q.w), 0x80402010u, hi);
    return (lo >> 7) | (hi << 1);
}

struct SamArgs {
    const uint8_t *chunk;
    const int64_t *starts;
    const int32_t *lens;
    int64_t n_lines;
    int64_t *fields;
    int64_t *status;
};

__global__ void __launch_bounds__(kSamThreads) sam_columns_kernel(const __grid_constant__ SamArgs a) {
    __shared__ int32_t s_tab[kSamWarps][kSamTabs + 1];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    int32_t *tab = s_tab[warp];
    // a '\r' that ends a line is not part of its last column when the first line ends in one (as K10's columns)
    const int32_t l0 = a.lens[0];
    const bool cr = l0 > 0 && __ldg(a.chunk + a.starts[0] + l0 - 1) == '\r';
    const int64_t R = a.n_lines;
    for (int64_t r = ((int64_t)blockIdx.x * kSamThreads + threadIdx.x) / 32; r < R;
         r += (int64_t)gridDim.x * kSamWarps) {
        const int64_t s = a.starts[r];
        int32_t L = a.lens[r];
        const uint8_t *line = a.chunk + s;
        if (cr && L > 0 && __ldg(line + L - 1) == '\r') --L;
        const uintptr_t p0 = reinterpret_cast<uintptr_t>(line), p1 = p0 + (uintptr_t)L;
        int n_tabs = 0;
        for (uintptr_t w = p0 & ~(uintptr_t)15; w < p1 && n_tabs < kSamTabs; w += 512) {
            const uintptr_t u = w + 16 * (uintptr_t)lane;
            uint32_t m = 0;
            if (u < p1) {
                m = tab_mask16(__ldg(reinterpret_cast<const uint4 *>(u)));
                if (u < p0) m &= 0xFFFFu << (p0 - u);
                if (p1 - u < 16) m &= (1u << (p1 - u)) - 1;
            }
            const int cnt = __popc(m);
            int inc = cnt;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const int t = __shfl_up_sync(0xffffffffu, inc, o);
                if (lane >= o) inc += t;
            }
            for (int t = n_tabs + inc - cnt; m && t < kSamTabs; ++t, m &= m - 1)
                tab[t] = (int32_t)(u + __ffs(m) - 1 - p0);
            n_tabs += __shfl_sync(0xffffffffu, inc, 31);
        }
        __syncwarp();
        n_tabs = min(n_tabs, kSamTabs);
        int64_t *f = a.fields + r;
        if (n_tabs < kSamTabs - 1) {
            // fewer than 11 columns: a fault, and every field of the row is empty
            if (lane < BNPK_SAM_FIELDS) f[lane * R] = (lane & 1) || lane >= BNPK_SAM_F_FLAG ? 0 : s;
            if (lane == 0) report_fault(a.status, fault_column(r, n_tabs + 1, BNPK_BAD_COLUMNS));
        } else if (lane < kSamTabs) {
            const int32_t f0 = lane ? tab[lane - 1] + 1 : 0, f1 = lane < n_tabs ? tab[lane] : L;
            const int text = kColStart[lane];
            if (text >= 0) {
                f[text * R] = s + f0;
                f[(text + 1) * R] = f1 - f0;
            } else {
                // an optional sign and 1 to 18 digits (as K10's integer columns)
                const int32_t n = f1 - f0;
                const uint8_t c0 = n > 0 ? __ldg(line + f0) : (uint8_t)0;
                const int sign = c0 == '-' || c0 == '+';
                bool ok = n > sign && n - sign <= kMaxDigits;
                int64_t v = 0;
                for (int32_t i = f0 + sign; ok && i < f1; ++i) {
                    const unsigned d = (unsigned)__ldg(line + i) - '0';
                    ok = d < 10;
                    v = v * 10 + d;
                }
                f[kColValue[lane] * R] = ok ? (c0 == '-' ? -v : v) : 0;
                if (!ok) report_fault(a.status, fault_column(r, lane, BNPK_BAD_INT));
            }
        } else if (lane == kSamTabs) {
            const int32_t e0 = n_tabs == kSamTabs ? tab[kSamTabs - 1] + 1 : L;
            f[BNPK_SAM_F_EXTRA_START * R] = s + e0;
            f[BNPK_SAM_F_EXTRA_LEN * R] = L - e0;
        }
        __syncwarp();       // the next line's walk overwrites the tab offsets
    }
}

// the CigarOpEncoding code of a CIGAR op letter (its index in "MIDNSHP=X"), or -1
__device__ __forceinline__ int cigar_code(uint32_t c) {
    switch (c) {
        case 'M': return 0;
        case 'I': return 1;
        case 'D': return 2;
        case 'N': return 3;
        case 'S': return 4;
        case 'H': return 5;
        case 'P': return 6;
        case '=': return 7;
        case 'X': return 8;
    }
    return -1;
}

struct CigarArgs {
    const uint8_t *base;
    const int64_t *starts;
    const int32_t *lens;
    int64_t n_rows;
    int32_t *counts;
    int64_t *ref_len;
    const int64_t *offsets;
    uint8_t *op;
    int64_t *length;
    int64_t *status;
};

// Walks the CIGAR text of row r: `*`, or ops of 1 to 9 digits and a letter of MIDNSHP=X.  UNPACK writes at most
// `room` ops from op/length; without it the op count and the reference length are returned.  False for invalid text.
template <bool UNPACK>
__device__ __forceinline__ bool walk_cigar(const uint8_t *p, int32_t L, int64_t room, uint8_t *op, int64_t *length,
                                           int32_t &n_ops, int64_t &ref_len) {
    n_ops = 0;
    ref_len = 0;
    if (L == 1 && __ldg(p) == '*') return true;
    int64_t v = 0;
    int nd = 0;
    for (int32_t i = 0; i < L; ++i) {
        const uint32_t c = __ldg(p + i);
        const unsigned d = c - '0';
        if (d < 10) {
            v = v * 10 + d;
            if (++nd > kMaxCigarDigits) return false;
            continue;
        }
        const int code = cigar_code(c);
        if (code < 0 || nd == 0) return false;
        if constexpr (UNPACK) {
            if (n_ops < room) {
                op[n_ops] = (uint8_t)code;
                length[n_ops] = v;
            }
        } else {
            // M (0), D (2), N (3), = (7) and X (8) consume the reference
            if ((0x18du >> code) & 1) ref_len += v;
        }
        ++n_ops;
        v = 0;
        nd = 0;
    }
    return nd == 0 && n_ops > 0;
}

__global__ void __launch_bounds__(256) cigar_count_kernel(const __grid_constant__ CigarArgs a) {
    for (int64_t r = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; r < a.n_rows; r += (int64_t)gridDim.x * blockDim.x) {
        const int32_t L = max(a.lens[r], 0);
        int32_t n_ops;
        int64_t ref_len;
        const bool ok = walk_cigar<false>(a.base + a.starts[r], L, 0, nullptr, nullptr, n_ops, ref_len);
        a.counts[r] = ok ? n_ops : 0;
        a.ref_len[r] = ok ? ref_len : 0;
        if (!ok) report_fault(a.status, fault_column(r, 5, BNPK_BAD_CIGAR));
    }
}

__global__ void __launch_bounds__(256) cigar_unpack_kernel(const __grid_constant__ CigarArgs a) {
    for (int64_t r = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; r < a.n_rows; r += (int64_t)gridDim.x * blockDim.x) {
        const int64_t o = a.offsets[r], room = a.offsets[r + 1] - o;
        if (room <= 0) continue;
        int32_t n_ops;
        int64_t unused;
        walk_cigar<true>(a.base + a.starts[r], max(a.lens[r], 0), room, a.op + o, a.length + o, n_ops, unused);
    }
}

}  // namespace

}  // namespace bnpk

using namespace bnpk;

extern "C" {

int bnpk_sam_columns(const uint8_t *chunk, size_t /* n: the lines lie inside it */, const int64_t *line_starts,
                     const int32_t *line_lens, size_t n_lines, int64_t *fields, int64_t *status, void *stream) {
    if (n_lines == 0) return 0;
    if (!chunk || !line_starts || !line_lens || !fields || !status)
        return set_err(BNPK_E_BADARG, "chunk, line_starts, line_lens, fields and status are required");
    const SamArgs a{chunk, line_starts, line_lens, (int64_t)n_lines, fields, status};
    return launch("sam_columns_kernel", sam_columns_kernel, grid_cap((n_lines + kSamWarps - 1) / kSamWarps, 8),
                  kSamThreads, 0, (cudaStream_t)stream, false, a);
}

int bnpk_cigar_count(const uint8_t *base, size_t /* base_bytes */, const int64_t *starts, const int32_t *lens,
                     size_t n_rows, int32_t *counts, int64_t *ref_len, int64_t *status, void *stream) {
    if (n_rows == 0) return 0;
    if (!base || !starts || !lens || !counts || !ref_len || !status)
        return set_err(BNPK_E_BADARG, "base, starts, lens, counts, ref_len and status are required");
    const CigarArgs a{base, starts, lens, (int64_t)n_rows, counts, ref_len, nullptr, nullptr, nullptr, status};
    return launch("cigar_count_kernel", cigar_count_kernel, grid_cap((n_rows + 255) / 256, 8), 256, 0,
                  (cudaStream_t)stream, false, a);
}

int bnpk_cigar_unpack(const uint8_t *base, size_t /* base_bytes */, const int64_t *starts, const int32_t *lens,
                      size_t n_rows, const int64_t *offsets, uint8_t *op, int64_t *length, void *stream) {
    if (n_rows == 0) return 0;
    if (!base || !starts || !lens || !offsets || !op || !length)
        return set_err(BNPK_E_BADARG, "base, starts, lens, offsets, op and length are required");
    const CigarArgs a{base, starts, lens, (int64_t)n_rows, nullptr, nullptr, offsets, op, length, nullptr};
    return launch("cigar_unpack_kernel", cigar_unpack_kernel, grid_cap((n_rows + 255) / 256, 8), 256, 0,
                  (cudaStream_t)stream, false, a);
}

}  // extern "C"
