// track_kernels.cu -- float64 signal tracks on the device: decimal text to double (bedGraph values), and the reductions
// and operators of float64 run-length tracks (FloatRunLengthArray, arithmetics/intervals.py).
//
// parse_float_kernel: one thread per row of text.  The grammar is checked and the significand gathered into a uint64
//   of at most 19 significant digits; the value is then exact by Clinger's fast path (at most 15 digits, |exp10| <= 22:
//   one correctly rounded multiply or divide by an exact power of ten) or by Eisel-Lemire with a 128-bit product of
//   the normalised significand and a truncated power of five from a host-built table (no fallback is needed for
//   significands below 2^64: Mushtak & Lemire, "Fast number parsing without fallback", 2023).
// track_f64_locate_kernel / track_f64_scan_kernel / track_f64_reduce_kernel / track_f64_fold_kernel: the flat list of
//   (query, run) pairs of bnpk_runs_reduce, cut into chunks whose size depends only on the list's length.  A query that
//   lies in one chunk is reduced by one thread in run order; a longer one leaves one partial per chunk, and one warp
//   folds its partials in chunk order (lane l takes chunks l, l + 32, ..., then a fixed butterfly).  No atomics: a sum
//   has the same bits on every run, whatever the grid.
// track_f64_combine_kernel: the merge path of runs_combine_kernel over float64 values; a run starts where the value's
//   bits change, so the output is canonical under bitwise equality.
#include <cmath>

#include "bnpk_host.h"

namespace bnpk {

namespace {

constexpr int kMaxSigDigits = 19;          // significant digits of a parsed value: the significand fits a uint64
constexpr int kClingerDigits = 15;
constexpr int kPow5Min = -342, kPow5Max = 308;
constexpr int kWalkItems = 16;             // (query, run) pairs of a reduction chunk, at least
constexpr int64_t kExpCap = 100000;        // an exponent this large already over- or underflows

__device__ __constant__ const double kPow10[23] = {1e0,  1e1,  1e2,  1e3,  1e4,  1e5,  1e6,  1e7,
                                                   1e8,  1e9,  1e10, 1e11, 1e12, 1e13, 1e14, 1e15,
                                                   1e16, 1e17, 1e18, 1e19, 1e20, 1e21, 1e22};

// --------------------------------------------------------------------------------------------------------------------
// decimal text to double
// --------------------------------------------------------------------------------------------------------------------
// The IEEE binary64 bits of w * 10^q, correctly rounded (half to even), for 0 < w < 2^64 (Eisel-Lemire).  pow5 holds
// (high, low) words of the truncated 128-bit 5^q for q in [kPow5Min, kPow5Max].
__device__ __forceinline__ uint64_t eisel_lemire(uint64_t w, int q, const uint64_t *pow5) {
    if (q < kPow5Min) return 0;
    if (q > kPow5Max) return 0x7FFull << 52;
    const int lz = __clzll((long long)w);
    w <<= lz;
    const uint64_t *t = pow5 + 2 * (q - kPow5Min);
    const uint64_t t_hi = __ldg(t), t_lo = __ldg(t + 1);
    uint64_t hi = __umul64hi(w, t_hi), lo = w * t_hi;
    if ((hi & 0x1FF) == 0x1FF) {
        // the truncated product may be off in the bits that decide the rounding: add the next 64 bits of the power
        const uint64_t s_hi = __umul64hi(w, t_lo);
        lo += s_hi;
        if (s_hi > lo) ++hi;
    }
    const int upper = (int)(hi >> 63);
    const int shift = upper + 64 - 52 - 3;
    uint64_t m = hi >> shift;
    int p2 = ((((152170 + 65536) * q) >> 16) + 63) + upper - lz + 1023;
    if (p2 <= 0) {
        // subnormal or zero
        if (-p2 + 1 >= 64) return 0;
        m >>= -p2 + 1;
        m += m & 1;
        m >>= 1;
        p2 = m < (1ull << 52) ? 0 : 1;
        return (uint64_t)p2 << 52 | (m & ((1ull << 52) - 1));
    }
    // exactly half way between two doubles: round to even
    if (lo <= 1 && q >= -4 && q <= 23 && (m & 3) == 1 && (m << shift) == hi) m &= ~1ull;
    m += m & 1;
    m >>= 1;
    if (m >= (2ull << 52)) {
        m = 1ull << 52;
        ++p2;
    }
    m &= ~(1ull << 52);
    if (p2 >= 0x7FF) return 0x7FFull << 52;
    return (uint64_t)p2 << 52 | m;
}

// [+-]? (digits ['.' digits?] | '.' digits) ([eE] [+-]? digits)? of at most 19 significant digits: its double's bits
// in `bits`, or false.
__device__ __forceinline__ bool parse_decimal(const uint8_t *p, int32_t L, const uint64_t *pow5, uint64_t &bits) {
    int32_t i = 0;
    bool neg = false;
    if (i < L) {
        const uint32_t c = __ldg(p);
        if (c == '+' || c == '-') {
            neg = c == '-';
            ++i;
        }
    }
    uint64_t w = 0;                 // the digits from the first to the last non-zero one
    int nd = 0, pending = 0;        // digits in w; zeros after w's last digit
    int64_t n_digits = 0, n_frac = 0;
    bool frac = false;
    for (; i < L; ++i) {
        const uint32_t c = __ldg(p + i);
        const unsigned d = c - '0';
        if (d >= 10) {
            if (c == '.' && !frac) {
                frac = true;
                continue;
            }
            break;
        }
        ++n_digits;
        n_frac += frac;
        if (d == 0) {
            pending += nd > 0;
            continue;
        }
        nd += pending + 1;
        if (nd > kMaxSigDigits) return false;
        for (; pending; --pending) w *= 10;
        w = w * 10 + d;
    }
    if (n_digits == 0) return false;
    int64_t e = 0;
    if (i < L && (__ldg(p + i) | 0x20) == 'e') {
        ++i;
        bool e_neg = false;
        if (i < L) {
            const uint32_t c = __ldg(p + i);
            if (c == '+' || c == '-') {
                e_neg = c == '-';
                ++i;
            }
        }
        int32_t ne = 0;
        for (; i < L; ++i) {
            const unsigned d = (uint32_t)__ldg(p + i) - '0';
            if (d >= 10) break;
            ++ne;
            if (e < kExpCap) e = e * 10 + d;
        }
        if (ne == 0) return false;
        if (e_neg) e = -e;
    }
    if (i != L) return false;
    const uint64_t sign = (uint64_t)neg << 63;
    if (w == 0) {
        bits = sign;
        return true;
    }
    int64_t q64 = e + pending - n_frac;
    q64 = max(min(q64, (int64_t)kPow5Max + 1), (int64_t)kPow5Min - 1);
    const int q = (int)q64;
    if (nd <= kClingerDigits && q >= -22 && q <= 22) {
        // Clinger: w and 10^|q| are exact doubles, so one correctly rounded operation gives the answer
        const double v = q < 0 ? __ddiv_rn((double)w, kPow10[-q]) : __dmul_rn((double)w, kPow10[q]);
        bits = (uint64_t)__double_as_longlong(v) | sign;
        return true;
    }
    bits = eisel_lemire(w, q, pow5) | sign;
    return true;
}

struct ParseArgs {
    const uint8_t *base;
    const int64_t *starts;
    const int32_t *lens;
    int64_t n_rows;
    int column;
    const uint64_t *pow5;
    double *out;
    int64_t *status;
};

__global__ void __launch_bounds__(256) parse_float_kernel(const __grid_constant__ ParseArgs a) {
    for (int64_t r = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; r < a.n_rows; r += (int64_t)gridDim.x * blockDim.x) {
        uint64_t bits = 0;
        const bool ok = parse_decimal(a.base + a.starts[r], max(a.lens[r], 0), a.pow5, bits);
        a.out[r] = __longlong_as_double((long long)(ok ? bits : 0));
        if (!ok) report_fault(a.status, fault_column(r, a.column, BNPK_BAD_FLOAT));
    }
}

// --------------------------------------------------------------------------------------------------------------------
// reductions over float64 runs
// --------------------------------------------------------------------------------------------------------------------
// first index i in [lo, hi) with a[i] > x (hi if none)
__device__ __forceinline__ int64_t first_above(const int64_t *a, int64_t lo, int64_t hi, int64_t x) {
    while (lo < hi) {
        const int64_t mid = (lo + hi) >> 1;
        if (a[mid] <= x) lo = mid + 1;
        else hi = mid;
    }
    return lo;
}

// first index i in [lo, hi) with a[i] >= x (hi if none)
__device__ __forceinline__ int64_t first_at_least(const int64_t *a, int64_t lo, int64_t hi, int64_t x) {
    while (lo < hi) {
        const int64_t mid = (lo + hi) >> 1;
        if (a[mid] < x) lo = mid + 1;
        else hi = mid;
    }
    return lo;
}

struct F64RunArgs {
    const int64_t *starts;       // int64[R + 1]
    const double *values;        // double[R]
    int64_t n_runs;
    const int64_t *q_start, *q_stop;
    int64_t n_q;
    int mode;
    int64_t *first, *count, *offs;   // per query: first run, runs overlapped, exclusive scan of count (int64[n_q + 1])
    double *partial;                 // two per chunk: the chunk's first and last piece of a query that crosses it
    int64_t n_chunks_cap;            // the chunks are at least kWalkItems pairs and at most this many
    double *out;
};

__device__ __forceinline__ double f64_identity(int mode) {
    return mode == BNPK_RUNS_MAX ? -INFINITY : mode == BNPK_RUNS_MIN ? INFINITY : 0.0;
}

// NaN wins; of two equal values the larger (max) / smaller (min) sign of zero wins, so the result has one bit pattern
// whatever the order
__device__ __forceinline__ double f64_reduce(int mode, double acc, double v) {
    switch (mode) {
        case BNPK_RUNS_MAX:
            if (isnan(acc) || isnan(v)) return isnan(acc) ? acc : v;
            return acc > v ? acc : v > acc ? v : (signbit(acc) ? v : acc);
        case BNPK_RUNS_MIN:
            if (isnan(acc) || isnan(v)) return isnan(acc) ? acc : v;
            return acc < v ? acc : v < acc ? v : (signbit(acc) ? acc : v);
        case BNPK_RUNS_SUM: return acc + v;
        default: return (acc != 0.0 || v != 0.0 || isnan(v)) ? 1.0 : 0.0;
    }
}

__device__ __forceinline__ void f64_query_range(const F64RunArgs &a, int64_t q, int64_t &s, int64_t &e) {
    const int64_t size = a.starts[a.n_runs];
    s = min(max(a.q_start[q], (int64_t)0), size);
    e = min(max(a.q_stop[q], s), size);
}

// the (query, run) pairs per chunk: a function of the list's length alone
__device__ __forceinline__ int64_t chunk_items(int64_t total, int64_t cap) {
    return max((int64_t)kWalkItems, (total + cap - 1) / cap);
}

__global__ void __launch_bounds__(256) track_f64_locate_kernel(const __grid_constant__ F64RunArgs a) {
    for (int64_t q = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; q < a.n_q; q += (int64_t)gridDim.x * blockDim.x) {
        int64_t s, e;
        f64_query_range(a, q, s, e);
        const int64_t r0 = max(first_above(a.starts, 0, a.n_runs, s) - 1, (int64_t)0);
        a.first[q] = r0;
        a.count[q] = e > s ? first_at_least(a.starts, r0, a.n_runs, e) - r0 : 0;
        a.out[q] = f64_identity(a.mode);
    }
}

__global__ void __launch_bounds__(kScanThreads) track_f64_scan_kernel(const int64_t *count, int64_t n, int64_t *offs,
                                                                      uint64_t *ws) {
    exclusive_offsets(n, offs, ws, [&](int64_t i) { return (uint64_t)count[i]; });
}

// One thread per chunk [c * C, (c + 1) * C) of the pair list.  A piece of a query that the chunk holds whole goes to
// out; a piece that began in an earlier chunk to partial[2c], one that goes on into a later chunk to partial[2c + 1].
__global__ void __launch_bounds__(256) track_f64_reduce_kernel(const __grid_constant__ F64RunArgs a) {
    const int64_t total = a.offs[a.n_q];
    const int64_t C = chunk_items(total, a.n_chunks_cap);
    const int64_t n_chunks = (total + C - 1) / C;
    for (int64_t c = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; c < n_chunks; c += (int64_t)gridDim.x * blockDim.x) {
        const int64_t w0 = c * C, w1 = min(w0 + C, total);
        int64_t q = first_above(a.offs, 0, a.n_q + 1, w0) - 1;
        int64_t s, e;
        f64_query_range(a, q, s, e);
        double acc = f64_identity(a.mode);
        for (int64_t w = w0; w < w1; ++w) {
            if (w >= a.offs[q + 1]) {
                // the piece of q ends inside the chunk
                if (a.offs[q] >= w0) a.out[q] = acc;
                else a.partial[2 * c] = acc;
                acc = f64_identity(a.mode);
                do ++q; while (w >= a.offs[q + 1]);
                f64_query_range(a, q, s, e);
            }
            const int64_t r = a.first[q] + (w - a.offs[q]);
            const double v = a.values[r];
            const double x = a.mode == BNPK_RUNS_SUM ? v * (double)(min(a.starts[r + 1], e) - max(a.starts[r], s)) : v;
            acc = f64_reduce(a.mode, acc, x);
        }
        const bool began_here = a.offs[q] >= w0, ends_here = a.offs[q + 1] <= w1;
        if (began_here && ends_here) a.out[q] = acc;
        else if (!began_here) a.partial[2 * c] = acc;
        else a.partial[2 * c + 1] = acc;
    }
}

// One warp per query that crosses a chunk border: its partials folded in chunk order.
__global__ void __launch_bounds__(256) track_f64_fold_kernel(const __grid_constant__ F64RunArgs a) {
    const int64_t total = a.offs[a.n_q];
    const int64_t C = chunk_items(total, a.n_chunks_cap);
    const int lane = threadIdx.x & 31;
    const int64_t warps = (int64_t)gridDim.x * (blockDim.x / 32);
    for (int64_t q = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) / 32; q < a.n_q; q += warps) {
        const int64_t o0 = a.offs[q], o1 = a.offs[q + 1];
        if (o1 == o0) continue;
        const int64_t c0 = o0 / C, c1 = (o1 - 1) / C;
        if (c0 == c1) continue;
        double acc = f64_identity(a.mode);
        for (int64_t c = c0 + lane; c <= c1; c += 32)
            acc = f64_reduce(a.mode, acc, a.partial[c == c0 ? 2 * c + 1 : 2 * c]);
#pragma unroll
        for (int o = 16; o; o >>= 1) acc = f64_reduce(a.mode, acc, __shfl_xor_sync(0xffffffffu, acc, o));
        if (lane == 0) a.out[q] = acc;
    }
}

// --------------------------------------------------------------------------------------------------------------------
// two float64 tracks into one
// --------------------------------------------------------------------------------------------------------------------
// NumPy's element rules: minimum / maximum give a NaN operand, else the second operand unless the first is strictly
// smaller / larger; comparisons give 1.0 or 0.0.
__device__ __forceinline__ double apply_f64(int op, double a, double b) {
    switch (op) {
        case BNPK_OP_ADD: return a + b;
        case BNPK_OP_SUB: return a - b;
        case BNPK_OP_MUL: return a * b;
        case BNPK_OP_DIV: return __ddiv_rn(a, b);
        case BNPK_OP_MIN: return (isnan(a) || a < b) ? a : b;
        case BNPK_OP_MAX: return (isnan(a) || a > b) ? a : b;
        case BNPK_OP_EQ: return a == b;
        case BNPK_OP_NE: return a != b;
        case BNPK_OP_LT: return a < b;
        case BNPK_OP_LE: return a <= b;
        case BNPK_OP_GT: return a > b;
        default: return a >= b;
    }
}

__device__ __forceinline__ int64_t bits_of(double v) { return (int64_t)__double_as_longlong(v); }

struct F64CombineArgs {
    const int64_t *a_starts, *b_starts;     // a_starts[n_a] = b_starts[n_b] = the size
    const double *a_values, *b_values;
    int64_t n_a, n_b;
    int op;
    int64_t *out_starts;
    double *out_values;
    int64_t *n_out;
    uint64_t *ws;
};

__global__ void __launch_bounds__(kScanThreads) track_f64_combine_kernel(const __grid_constant__ F64CombineArgs a) {
    __shared__ ScanSmem sm;
    const int64_t n = a.n_a + a.n_b;
    const int64_t n_tiles = (n + kScanTile - 1) / kScanTile;
    const int64_t *as = a.a_starts, *bs = a.b_starts;
    for (int64_t tile; (tile = next_tile(a.ws, n_tiles, sm)) >= 0;) {
        const int64_t i0 = tile * kScanTile + (int64_t)threadIdx.x * kScanItems;
        // the merged starts before i0: ia of A's and i0 - ia of B's, an A start before a B start at the same position
        const int64_t d = min(i0, n);
        int64_t lo = max(d - a.n_b, (int64_t)0), hi = min(d, a.n_a);
        while (lo < hi) {
            const int64_t mid = (lo + hi) >> 1;
            if (as[mid] <= bs[d - 1 - mid]) lo = mid + 1;
            else hi = mid;
        }
        int64_t ia = lo, ib = d - lo;
        int64_t pos[kScanItems];
        double val[kScanItems];
        uint32_t emit = 0;
#pragma unroll
        for (int j = 0; j < kScanItems; ++j) {
            if (i0 + j >= n) break;
            int64_t p, ja, jb;
            bool last;
            if (as[ia] <= bs[ib]) {
                p = as[ia++];
                last = bs[ib] != p;
                ja = ia - 1;
                jb = ib;
            } else {
                p = bs[ib++];
                last = true;
                ja = ia - (ia > 0 && as[ia - 1] == p);
                jb = ib - 1;
            }
            if (!last) continue;
            const double v = apply_f64(a.op, a.a_values[ia - 1], a.b_values[ib - 1]);
            if (p == 0 || bits_of(v) != bits_of(apply_f64(a.op, a.a_values[ja - 1], a.b_values[jb - 1]))) {
                emit |= 1u << j;
                pos[j] = p;
                val[j] = v;
            }
        }
        uint64_t o = block_exclusive<Sum>((uint64_t)__popc(emit), tile, a.ws + kWsHeaderWords, sm);
#pragma unroll
        for (int j = 0; j < kScanItems; ++j) {
            if (emit >> j & 1) {
                a.out_starts[o] = pos[j];
                a.out_values[o] = val[j];
                ++o;
            }
        }
        if (tile == n_tiles - 1 && threadIdx.x == kScanThreads - 1) {
            a.n_out[0] = (int64_t)o;
            a.out_starts[o] = as[a.n_a];
        }
    }
}

}  // namespace
}  // namespace bnpk

using namespace bnpk;

extern "C" {

int bnpk_parse_float(const uint8_t *base, size_t /* base_bytes: the rows lie inside it */, const int64_t *starts,
                     const int32_t *lens, size_t n_rows, int column, const uint64_t *pow5_table, double *out,
                     int64_t *status, void *stream) {
    if (column < 0 || column > 31) return set_err(BNPK_E_BADARG, "column must be in [0, 31]");
    if (n_rows == 0) return 0;
    if (!base || !starts || !lens || !pow5_table || !out || !status)
        return set_err(BNPK_E_BADARG, "base, starts, lens, pow5_table, out and status are required");
    const ParseArgs a{base, starts, lens, (int64_t)n_rows, column, pow5_table, out, status};
    return launch("parse_float_kernel", parse_float_kernel, grid_cap((n_rows + 255) / 256, 8), 256, 0,
                  (cudaStream_t)stream, false, a);
}

int bnpk_track_f64_reduce(const int64_t *run_starts, const double *values, size_t n_runs, const int64_t *q_start,
                          const int64_t *q_stop, size_t n_q, int mode, double *out, int64_t *scratch, double *partial,
                          size_t n_chunks_cap, void *workspace, size_t workspace_bytes, void *stream) {
    if (mode < BNPK_RUNS_MAX || mode > BNPK_RUNS_ANY) return set_err(BNPK_E_BADARG, "unknown reduction");
    if (n_runs < 1 || !run_starts || !values) return set_err(BNPK_E_BADARG, "at least one run is required");
    if (n_chunks_cap < 1) return set_err(BNPK_E_BADARG, "n_chunks_cap must be at least 1");
    if (n_q == 0) return 0;
    if (!q_start || !q_stop || !out || !scratch || !partial || !workspace)
        return set_err(BNPK_E_BADARG, "q_start, q_stop, out, scratch, partial and workspace are required");
    cudaStream_t st = (cudaStream_t)stream;
    size_t n_tiles;
    if (int rc = scan_workspace(n_q, 1, workspace, workspace_bytes, st, n_tiles)) return rc;
    F64RunArgs a{run_starts, values, (int64_t)n_runs, q_start, q_stop, (int64_t)n_q, mode,
                 scratch, scratch + n_q, scratch + 2 * n_q, partial, (int64_t)n_chunks_cap, out};
    int rc = launch("track_f64_locate_kernel", track_f64_locate_kernel, grid_cap((n_q + 255) / 256, 8), 256, 0, st,
                    false, a);
    if (rc) return rc;
    rc = launch("track_f64_scan_kernel", track_f64_scan_kernel, grid_cap(n_tiles, 4), kScanThreads, 0, st, false,
                (const int64_t *)a.count, (int64_t)n_q, a.offs, (uint64_t *)workspace);
    if (rc) return rc;
    // the pair list is as long as the device says; the grid fills the GPU and strides over its chunks
    rc = launch("track_f64_reduce_kernel", track_f64_reduce_kernel, grid_cap((size_t)-1, 8), 256, 0, st, false, a);
    if (rc) return rc;
    return launch("track_f64_fold_kernel", track_f64_fold_kernel, grid_cap((n_q + 7) / 8, 8), 256, 0, st, false, a);
}

int bnpk_track_f64_combine(const int64_t *a_starts, const double *a_values, size_t n_a, const int64_t *b_starts,
                           const double *b_values, size_t n_b, int op, int64_t *out_starts, double *out_values,
                           int64_t *n_out, void *workspace, size_t workspace_bytes, void *stream) {
    const bool known = op == BNPK_OP_ADD || op == BNPK_OP_SUB || op == BNPK_OP_MUL || op == BNPK_OP_DIV ||
                       (op >= BNPK_OP_MIN && op <= BNPK_OP_GE);
    if (!known) return set_err(BNPK_E_BADARG, "unknown float track operator");
    if (!a_starts || !b_starts || !out_starts || !n_out || !workspace)
        return set_err(BNPK_E_BADARG, "a_starts, b_starts, out_starts, n_out and workspace are required");
    if ((n_a == 0) != (n_b == 0)) return set_err(BNPK_E_BADARG, "a track without runs is empty: both must be");
    if (n_a && (!a_values || !b_values || !out_values))
        return set_err(BNPK_E_BADARG, "a_values, b_values and out_values are required");
    cudaStream_t st = (cudaStream_t)stream;
    if (n_a == 0) {
        BNPK_CUDA(cudaMemsetAsync(n_out, 0, sizeof(int64_t), st));
        BNPK_CUDA(cudaMemsetAsync(out_starts, 0, sizeof(int64_t), st));
        return 0;
    }
    size_t n_tiles;
    if (int rc = scan_workspace(n_a + n_b, 1, workspace, workspace_bytes, st, n_tiles)) return rc;
    F64CombineArgs a{a_starts, b_starts, a_values, b_values, (int64_t)n_a, (int64_t)n_b, op,
                     out_starts, out_values, n_out, (uint64_t *)workspace};
    return launch("track_f64_combine_kernel", track_f64_combine_kernel, grid_cap(n_tiles, 4), kScanThreads, 0, st,
                  false, a);
}

}  // extern "C"
