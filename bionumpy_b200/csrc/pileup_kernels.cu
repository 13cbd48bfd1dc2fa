// pileup_kernels.cu -- coverage runs, reductions and gathers over runs, interval merge and row equality on the device
// (get_pileup / get_boolean_mask / merge_intervals arithmetics/intervals.py:137-304, GenomicRunLengthArray and its
// indexing by intervals, genomic_data/genomic_track.py).
//
// interval_events_kernel: one thread per interval; checks it against its contig and writes its two event keys
//   (global position << 1 | 1 for a start, global position << 1 for a stop).
// pileup_runs_kernel: one single-pass decoupled look-back scan over the sorted event keys, 2048 keys per tile.  The
//   coverage after every key is an exclusive sum (look-back 1); a run starts at the last key of each group of equal
//   positions whose coverage differs from the coverage before the group's first key; the runs are compacted in order
//   (look-back 2).  A group that began in an earlier thread or tile has its start found by binary search on the keys.
// runs_locate_kernel / runs_reduce_kernel: the runs each query overlaps are counted and scanned, and the grid walks
//   the flat list of (query, run) pairs, 16 per thread, so that one long query and a million short ones both spread
//   over the whole GPU; partial results are combined with one atomic per thread and query (one per warp when the
//   whole warp is in one query).
// runs_extract_kernel: 16 consecutive output positions per thread, one run search per thread, then a walk.
// interval_merge_kernel: a segmented inclusive max-scan of stop (look-back 1 with an ordered segmented-max operator)
//   and the compaction of the first row of every group (look-back 2).
// rows_equal_prev_kernel: one thread per row, a full byte compare with the previous row.
// runs_combine_kernel: a merge path over the run starts of two tracks, 2048 merged starts per tile, each thread's first
//   split between the tracks found by binary search on its diagonal; every start decides alone whether a run of
//   op(a, b) begins there, and the runs are compacted in order (one look-back).
// interval_intersect_kernel: row r > 0 of a segment pairs with row r - 1 when stop[r - 1] > start[r]; the pairs are
//   compacted in order (one look-back) and their overlaps summed (one atomic per block and tile).
// runs_to_intervals_kernel: 8 runs per thread; two binary searches of the contig ends (in shared memory when they fit)
//   give each run's pieces, and the rows they open are compacted in order (one look-back).
#include "bnpk_host.h"

namespace bnpk {

namespace {

constexpr int kWalkItems = 16;
constexpr uint64_t kBias = 1ull << 59;          // merge: stop + kBias in [0, 2^60)
constexpr uint64_t kReset = 1ull << 61;         // merge: "a segment starts here" in the scanned word
constexpr int64_t kMaxPos = (int64_t)1 << 59;   // positions are in [0, 2^59)

// the value of a 62-bit look-back word as a signed number
__device__ __forceinline__ int64_t signed62(uint64_t v) { return (int64_t)(v << 2) >> 2; }

// first index i in [lo, hi) with a[i] >= x (hi if none)
__device__ __forceinline__ int64_t lower_bound(const int64_t *a, int64_t lo, int64_t hi, int64_t x) {
    while (lo < hi) {
        const int64_t mid = (lo + hi) >> 1;
        if (a[mid] < x) lo = mid + 1;
        else hi = mid;
    }
    return lo;
}

// first index i in [lo, hi) with a[i] > x (hi if none)
__device__ __forceinline__ int64_t upper_bound(const int64_t *a, int64_t lo, int64_t hi, int64_t x) {
    while (lo < hi) {
        const int64_t mid = (lo + hi) >> 1;
        if (a[mid] <= x) lo = mid + 1;
        else hi = mid;
    }
    return lo;
}

// --------------------------------------------------------------------------------------------------------------------
// events
// --------------------------------------------------------------------------------------------------------------------
struct EventArgs {
    const int64_t *start, *stop;
    const int32_t *ids;
    const int64_t *c_offset, *c_len;
    int64_t n_contigs, size, n_rows;
    int64_t *keys, *g_start, *g_stop, *status;
};

__global__ void __launch_bounds__(256) interval_events_kernel(const __grid_constant__ EventArgs a) {
    for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < a.n_rows; r += (int64_t)gridDim.x * blockDim.x) {
        const int64_t s = a.start[r], e = a.stop[r];
        int64_t off = 0, len = a.size;
        bool skip = false, ok = true;
        if (a.ids) {
            const int32_t id = a.ids[r];
            ok = id >= 0 && id < a.n_contigs;
            if (ok) {
                off = a.c_offset[id];
                len = a.c_len[id];
                skip = off < 0;             // a contig the caller leaves out: its rows are not checked and add nothing
            }
        }
        ok = skip || (ok && s >= 0 && e >= s && e <= len && off + len <= kMaxPos);
        const bool live = ok && !skip;
        if (a.keys) {
            a.keys[2 * r] = live ? (off + s) << 1 | 1 : 1;       // a bad or left-out row: an empty interval at 0
            a.keys[2 * r + 1] = live ? (off + e) << 1 : 0;
        }
        if (a.g_start) a.g_start[r] = live ? off + s : 0;
        if (a.g_stop) a.g_stop[r] = live ? off + e : 0;
        if (!ok) report_fault(a.status, r);
    }
}

// --------------------------------------------------------------------------------------------------------------------
// runs from sorted events
// --------------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kScanThreads) pileup_runs_kernel(const int64_t *keys, int64_t n, int64_t size,
                                                                   int any_mode, int64_t *run_starts,
                                                                   int64_t *run_values, int64_t *n_runs, uint64_t *ws) {
    __shared__ ScanSmem sm;
    const int tid = threadIdx.x;
    const int64_t n_tiles = n > 0 ? (n + kScanTile - 1) / kScanTile : 1;
    uint64_t *cov_state = ws + kWsHeaderWords;
    uint64_t *run_state = cov_state + n_tiles;
    for (int64_t tile; (tile = next_tile(ws, n_tiles, sm)) >= 0;) {
        const int64_t i0 = tile * kScanTile + (int64_t)tid * kScanItems;
        int64_t k[kScanItems];
        int64_t dsum = 0;
#pragma unroll
        for (int j = 0; j < kScanItems; ++j) {
            k[j] = i0 + j < n ? keys[i0 + j] : INT64_MAX;
            if (i0 + j < n) dsum += (k[j] & 1) ? 1 : -1;
        }
        const int64_t prev_pos = i0 > 0 && i0 <= n ? keys[i0 - 1] >> 1 : INT64_MIN;
        const int64_t next_pos = i0 + kScanItems < n ? keys[i0 + kScanItems] >> 1 : INT64_MAX;
        int64_t cov = signed62(block_exclusive<Sum>((uint64_t)dsum, tile, cov_state, sm));
        // the runs of this thread: where the coverage after a position's last key differs from the coverage before
        // its first key; position 0 always starts a run, and when no key is at 0, the run (0, 0) is the first
        int64_t val[kScanItems];
        uint32_t emit = 0;
        int64_t before = 0;
        bool before_known = false;
        const bool lead_zero = tile == 0 && tid == 0 && (n == 0 || (k[0] >> 1) != 0);
#pragma unroll
        for (int j = 0; j < kScanItems; ++j) {
            const int64_t i = i0 + j;
            if (i >= n) break;
            const int64_t pos = k[j] >> 1;
            if (pos != (j ? k[j - 1] >> 1 : prev_pos)) {
                before = cov;
                before_known = true;
            }
            cov += (k[j] & 1) ? 1 : -1;
            const int64_t nxt = j + 1 < kScanItems ? (i + 1 < n ? k[j + 1] >> 1 : INT64_MAX) : next_pos;
            if (nxt == pos || pos < 0 || pos >= size) continue;
            if (!before_known) {
                // the group began in an earlier thread or tile: its keys are [lo, i], stops before starts
                const int64_t lo = lower_bound(keys, 0, i + 1, pos << 1);
                const int64_t mid = lower_bound(keys, lo, i + 1, pos << 1 | 1);
                before = cov - ((i + 1 - mid) - (mid - lo));
            }
            const int64_t b = any_mode ? (int64_t)(before > 0) : before;
            const int64_t v = any_mode ? (int64_t)(cov > 0) : cov;
            if (pos == 0 || v != b) {
                emit |= 1u << j;
                val[j] = v;
            }
        }
        const uint64_t n_emit = (uint64_t)__popc(emit) + lead_zero;
        uint64_t o = block_exclusive<Sum>(n_emit, tile, run_state, sm);
        if (lead_zero) {
            run_starts[o] = 0;
            run_values[o] = 0;
            ++o;
        }
#pragma unroll
        for (int j = 0; j < kScanItems; ++j) {
            if (emit >> j & 1) {
                run_starts[o] = k[j] >> 1;
                run_values[o] = val[j];
                ++o;
            }
        }
        if (tile == n_tiles - 1 && tid == kScanThreads - 1) {
            // the last thread of the last tile: its exclusive prefix plus its own runs is every run
            n_runs[0] = (int64_t)o;
            run_starts[o] = size;      // the end of the last run
        }
    }
}

// --------------------------------------------------------------------------------------------------------------------
// reductions and gathers over runs
// --------------------------------------------------------------------------------------------------------------------
struct RunArgs {
    const int64_t *starts;       // int64[R + 1], starts[R] = the array's size
    const int64_t *values;       // int64[R]
    int64_t n_runs;
    const int64_t *q_start, *q_stop;
    int64_t n_q;
    int mode;
    int64_t *first, *count, *offs;   // per query: first run, runs overlapped, exclusive scan of count (int64[n_q + 1])
    int64_t *out;
};

__device__ __forceinline__ int64_t identity_of(int mode) {
    return mode == BNPK_RUNS_MAX ? INT64_MIN : mode == BNPK_RUNS_MIN ? INT64_MAX : 0;
}

// [a, b) of query q clipped to the array
__device__ __forceinline__ void query_range(const RunArgs &a, int64_t q, int64_t &s, int64_t &e) {
    const int64_t size = a.starts[a.n_runs];
    s = min(max(a.q_start[q], (int64_t)0), size);
    e = min(max(a.q_stop[q], s), size);
}

__global__ void __launch_bounds__(256) runs_locate_kernel(const __grid_constant__ RunArgs a) {
    for (int64_t q = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; q < a.n_q; q += (int64_t)gridDim.x * blockDim.x) {
        int64_t s, e;
        query_range(a, q, s, e);
        const int64_t r0 = max(upper_bound(a.starts, 0, a.n_runs, s) - 1, (int64_t)0);
        a.first[q] = r0;
        a.count[q] = e > s ? lower_bound(a.starts, r0, a.n_runs, e) - r0 : 0;
        a.out[q] = identity_of(a.mode);
    }
}

__global__ void __launch_bounds__(kScanThreads) count_scan_kernel(const int64_t *count, int64_t n, int64_t *offs,
                                                                  uint64_t *ws) {
    exclusive_offsets(n, offs, ws, [&](int64_t i) { return (uint64_t)count[i]; });
}

__device__ __forceinline__ int64_t combine(int mode, int64_t acc, int64_t v, int64_t overlap) {
    switch (mode) {
        case BNPK_RUNS_MAX: return max(acc, v);
        case BNPK_RUNS_MIN: return min(acc, v);
        case BNPK_RUNS_SUM: return (int64_t)((uint64_t)acc + (uint64_t)v * (uint64_t)overlap);
        default: return acc | (int64_t)(v != 0);
    }
}

__device__ __forceinline__ void flush(int mode, int64_t *out, int64_t v) {
    switch (mode) {
        case BNPK_RUNS_MAX: atomicMax((long long *)out, (long long)v); break;
        case BNPK_RUNS_MIN: atomicMin((long long *)out, (long long)v); break;
        case BNPK_RUNS_SUM: atomicAdd((unsigned long long *)out, (unsigned long long)v); break;
        default: if (v) atomicOr((unsigned long long *)out, 1ull); break;
    }
}

__device__ __forceinline__ int64_t warp_combine(int mode, int64_t v) {
#pragma unroll
    for (int o = 16; o; o >>= 1) {
        const int64_t t = __shfl_xor_sync(0xffffffffu, v, o);
        v = mode == BNPK_RUNS_MAX ? max(v, t) : mode == BNPK_RUNS_MIN ? min(v, t) :
            mode == BNPK_RUNS_SUM ? (int64_t)((uint64_t)v + (uint64_t)t) : (v | t);
    }
    return v;
}

__global__ void __launch_bounds__(256) runs_reduce_kernel(const __grid_constant__ RunArgs a) {
    const int64_t total = a.offs[a.n_q];
    const int64_t n_chunks = (total + kWalkItems - 1) / kWalkItems;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    // every lane runs the same number of rounds, so that the whole warp can meet at the flush
    const int64_t rounds = (n_chunks + stride - 1) / stride;
    const int64_t t0 = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    for (int64_t round = 0; round < rounds; ++round) {
        const int64_t w0 = (t0 + round * stride) * kWalkItems;
        int64_t q = -1, acc = identity_of(a.mode);
        if (w0 < total) {
            q = upper_bound(a.offs, 0, a.n_q + 1, w0) - 1;
            int64_t s, e;
            query_range(a, q, s, e);
            const int64_t w1 = min(w0 + kWalkItems, total);
            for (int64_t w = w0; w < w1; ++w) {
                if (w >= a.offs[q + 1]) {
                    flush(a.mode, a.out + q, acc);
                    acc = identity_of(a.mode);
                    do ++q; while (w >= a.offs[q + 1]);
                    query_range(a, q, s, e);
                }
                const int64_t r = a.first[q] + (w - a.offs[q]);
                const int64_t overlap = min(a.starts[r + 1], e) - max(a.starts[r], s);
                acc = combine(a.mode, acc, a.values[r], overlap);
            }
        }
        // the last query of every lane: one atomic per warp when the warp is in one query, else one per lane
        const unsigned same = __match_any_sync(0xffffffffu, q);
        if (same == 0xffffffffu) {
            acc = warp_combine(a.mode, acc);
            if ((threadIdx.x & 31) == 0 && q >= 0) flush(a.mode, a.out + q, acc);
        } else if (q >= 0) {
            flush(a.mode, a.out + q, acc);
        }
    }
}

struct ExtractArgs {
    const int64_t *starts;
    const int64_t *values;
    int64_t n_runs;
    const int64_t *q_start;
    int64_t n_q;
    const int64_t *out_offs;     // int64[n_q + 1]
    int64_t *out;
};

__global__ void __launch_bounds__(256) runs_extract_kernel(const __grid_constant__ ExtractArgs a) {
    const int64_t total = a.out_offs[a.n_q];
    const int64_t n_chunks = (total + kWalkItems - 1) / kWalkItems;
    for (int64_t c = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; c < n_chunks; c += (int64_t)gridDim.x * blockDim.x) {
        const int64_t o0 = c * kWalkItems, o1 = min(o0 + kWalkItems, total);
        int64_t q = upper_bound(a.out_offs, 0, a.n_q + 1, o0) - 1;
        int64_t pos = a.q_start[q] + (o0 - a.out_offs[q]);
        int64_t r = max(upper_bound(a.starts, 0, a.n_runs, pos) - 1, (int64_t)0);
        for (int64_t o = o0; o < o1; ++o, ++pos) {
            if (o >= a.out_offs[q + 1]) {
                do ++q; while (o >= a.out_offs[q + 1]);
                pos = a.q_start[q];
                r = max(upper_bound(a.starts, 0, a.n_runs, pos) - 1, (int64_t)0);
            }
            while (r + 1 < a.n_runs && pos >= a.starts[r + 1]) ++r;
            a.out[o] = a.values[r];
        }
    }
}

// --------------------------------------------------------------------------------------------------------------------
// merge
// --------------------------------------------------------------------------------------------------------------------
// The ordered segmented maximum of two scanned words, `before` and `after`: `after` alone when a segment starts in it.
struct SegMax {
    __device__ __forceinline__ static uint64_t combine(uint64_t before, uint64_t after) {
        return (after & kReset) ? after : (before & kReset) | max(before & ~kReset, after);
    }
};

struct MergeArgs {
    const int64_t *start, *stop;
    const uint8_t *same_prev;
    int64_t n, distance;
    int64_t *out_rows, *out_stops, *n_out, *status;
    uint64_t *ws;
};

__global__ void __launch_bounds__(kScanThreads) interval_merge_kernel(const __grid_constant__ MergeArgs a) {
    __shared__ ScanSmem sm;
    const int tid = threadIdx.x;
    const int64_t n_tiles = (a.n + kScanTile - 1) / kScanTile;
    uint64_t *max_state = a.ws + kWsHeaderWords;
    uint64_t *grp_state = max_state + n_tiles;
    const int64_t d = a.distance;
    for (int64_t tile; (tile = next_tile(a.ws, n_tiles, sm)) >= 0;) {
        const int64_t i0 = tile * kScanTile + (int64_t)tid * kScanItems;
        int64_t st[kScanItems + 1], sp[kScanItems];
        bool seg[kScanItems + 1];
        uint64_t agg = 0;
#pragma unroll
        for (int j = 0; j <= kScanItems; ++j) {
            const int64_t i = i0 + j;
            st[j] = i < a.n ? a.start[i] : 0;
            seg[j] = i >= a.n || i == 0 || (a.same_prev && !a.same_prev[i]);   // no flags: one segment
            if (j < kScanItems) {
                sp[j] = i < a.n ? a.stop[i] : 0;
                if (i < a.n) agg = SegMax::combine(agg, (seg[j] ? kReset : 0) | (uint64_t)(sp[j] + (int64_t)kBias));
            }
        }
        // the segmented max of the rows before this thread's first row
        uint64_t run = block_exclusive<SegMax>(agg, tile, max_state, sm);
        // running max before each row (within its segment), the group starts and ends
        const int64_t prev_start = i0 > 0 && i0 <= a.n ? a.start[i0 - 1] : 0;
        int64_t incl[kScanItems];
        uint32_t first = 0, last = 0;
#pragma unroll
        for (int j = 0; j < kScanItems; ++j) {
            const int64_t i = i0 + j;
            if (i >= a.n) break;
            const int64_t before = (int64_t)(run & ~kReset) - (int64_t)kBias;
            if (seg[j] || st[j] > before + d) first |= 1u << j;
            if (!seg[j] && st[j] < (j ? st[j - 1] : prev_start)) report_fault(a.status, i);
            run = SegMax::combine(run, (seg[j] ? kReset : 0) | (uint64_t)(sp[j] + (int64_t)kBias));
            incl[j] = (int64_t)(run & ~kReset) - (int64_t)kBias;
        }
#pragma unroll
        for (int j = 0; j < kScanItems; ++j) {
            const int64_t i = i0 + j;
            if (i >= a.n) break;
            if (seg[j + 1] || st[j + 1] > incl[j] + d) last |= 1u << j;
        }
        uint64_t g = block_exclusive<Sum>((uint64_t)__popc(first), tile, grp_state, sm);
#pragma unroll
        for (int j = 0; j < kScanItems; ++j) {
            if (first >> j & 1) a.out_rows[g++] = i0 + j;
            if (last >> j & 1) a.out_stops[g - 1] = incl[j];
        }
        if (tile == n_tiles - 1 && tid == kScanThreads - 1) a.n_out[0] = (int64_t)g;
    }
}

// --------------------------------------------------------------------------------------------------------------------
// row equality
// --------------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) rows_equal_prev_kernel(const uint8_t *base, const int64_t *starts,
                                                              const int32_t *lens, int64_t n_rows, uint8_t *flag) {
    for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < n_rows; r += (int64_t)gridDim.x * blockDim.x) {
        bool eq = r > 0 && lens[r] == lens[r - 1];
        if (eq) {
            const uint8_t *x = base + starts[r], *y = base + starts[r - 1];
            for (int32_t i = 0; i < lens[r] && eq; ++i) eq = x[i] == y[i];
        }
        flag[r] = eq;
    }
}

// --------------------------------------------------------------------------------------------------------------------
// two tracks into one
// --------------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ int64_t apply_op(int op, int64_t a, int64_t b) {
    const uint64_t x = (uint64_t)a, y = (uint64_t)b;
    switch (op) {
        case BNPK_OP_ADD: return (int64_t)(x + y);
        case BNPK_OP_SUB: return (int64_t)(x - y);
        case BNPK_OP_MUL: return (int64_t)(x * y);
        case BNPK_OP_AND: return a & b;
        case BNPK_OP_OR: return a | b;
        case BNPK_OP_XOR: return a ^ b;
        case BNPK_OP_MIN: return min(a, b);
        case BNPK_OP_MAX: return max(a, b);
        case BNPK_OP_EQ: return a == b;
        case BNPK_OP_NE: return a != b;
        case BNPK_OP_LT: return a < b;
        case BNPK_OP_LE: return a <= b;
        case BNPK_OP_GT: return a > b;
        default: return a >= b;
    }
}

struct CombineArgs {
    const int64_t *a_starts, *a_values;     // a_starts[n_a] = b_starts[n_b] = the size
    const int64_t *b_starts, *b_values;
    int64_t n_a, n_b;
    int op;
    int64_t *out_starts, *out_values, *n_out;
    uint64_t *ws;
};

__global__ void __launch_bounds__(kScanThreads) runs_combine_kernel(const __grid_constant__ CombineArgs a) {
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
        int64_t pos[kScanItems], val[kScanItems];
        uint32_t emit = 0;
#pragma unroll
        for (int j = 0; j < kScanItems; ++j) {
            if (i0 + j >= n) break;
            // the sizes at as[n_a] and bs[n_b] sort after every start, so neither track is read past its end
            int64_t p, ja, jb;
            bool last;
            if (as[ia] <= bs[ib]) {
                p = as[ia++];
                last = bs[ib] != p;                   // a B start at p comes next and closes the group
                ja = ia - 1;
                jb = ib;
            } else {
                p = bs[ib++];
                last = true;
                ja = ia - (ia > 0 && as[ia - 1] == p);
                jb = ib - 1;
            }
            if (!last) continue;
            // the value from p on, and the value at the previous start position (every track has a start at 0)
            const int64_t v = apply_op(a.op, a.a_values[ia - 1], a.b_values[ib - 1]);
            if (p == 0 || v != apply_op(a.op, a.a_values[ja - 1], a.b_values[jb - 1])) {
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

// --------------------------------------------------------------------------------------------------------------------
// intersect
// --------------------------------------------------------------------------------------------------------------------
struct IntersectArgs {
    const int64_t *start, *stop;
    const uint8_t *same_prev;
    int64_t n;
    int64_t *out_rows, *out_stops, *n_out, *overlap;
    uint64_t *ws;
};

__global__ void __launch_bounds__(kScanThreads) interval_intersect_kernel(const __grid_constant__ IntersectArgs a) {
    __shared__ ScanSmem sm;
    __shared__ uint64_t warp_overlap[kScanWarps];
    const int64_t n_tiles = (a.n + kScanTile - 1) / kScanTile;
    for (int64_t tile; (tile = next_tile(a.ws, n_tiles, sm)) >= 0;) {
        const int64_t i0 = tile * kScanTile + (int64_t)threadIdx.x * kScanItems;
        int64_t prev_stop = i0 > 0 && i0 <= a.n ? a.stop[i0 - 1] : 0;
        int64_t stops[kScanItems];
        uint32_t emit = 0;
        uint64_t over = 0;
#pragma unroll
        for (int j = 0; j < kScanItems; ++j) {
            const int64_t i = i0 + j;
            if (i >= a.n) break;
            const int64_t s = a.start[i];
            // row i pairs with row i - 1 of its segment when that row's (sorted) stop is past its start
            if (i > 0 && (!a.same_prev || a.same_prev[i]) && prev_stop > s) {
                emit |= 1u << j;
                stops[j] = prev_stop;
                over += (uint64_t)(prev_stop - s);
            }
            prev_stop = a.stop[i];
        }
        if (a.overlap) {
            over = warp_sum_u64(over);
            if ((threadIdx.x & 31) == 0) warp_overlap[threadIdx.x >> 5] = over;
        }
        uint64_t g = block_exclusive<Sum>((uint64_t)__popc(emit), tile, a.ws + kWsHeaderWords, sm);
        if (a.overlap && threadIdx.x == 0) {
            uint64_t total = 0;
#pragma unroll
            for (int w = 0; w < kScanWarps; ++w) total += warp_overlap[w];
            if (total) atomicAdd((unsigned long long *)a.overlap, (unsigned long long)total);
        }
        if (a.out_rows) {
#pragma unroll
            for (int j = 0; j < kScanItems; ++j) {
                if (emit >> j & 1) {
                    a.out_rows[g] = i0 + j;
                    a.out_stops[g] = stops[j];
                    ++g;
                }
            }
        } else {
            g += __popc(emit);
        }
        if (tile == n_tiles - 1 && threadIdx.x == kScanThreads - 1) a.n_out[0] = (int64_t)g;
    }
}

// --------------------------------------------------------------------------------------------------------------------
// runs -> interval rows
// --------------------------------------------------------------------------------------------------------------------
constexpr int kEndsSmem = 2048;     // contig ends staged in shared memory (16 KiB) when all C + 1 fit

struct ToIntervalsArgs {
    const int64_t *starts, *values;     // starts[n_runs] = the size = ends[n_contigs]
    int64_t n_runs;
    const int64_t *ends;                // int64[n_contigs + 1], strictly increasing from 0
    int64_t n_contigs;
    int all;
    int32_t *out_contig;
    int64_t *out_start, *out_stop, *out_value, *n_out;
    uint64_t *ws;
};

// Run i = [s, e) lies in contigs c .. c + pieces - 1, and the contig borders inside it cut it into `pieces` pieces.  In
// ALL mode every piece is a row.  In NONZERO mode a zero run has no piece, and a non-zero run's first piece continues
// the row of the run before unless s is a border or that run is zero ("opens"), its last piece leaves its row open
// for the next run unless e is a border or that run is zero ("closes").  So the rows are counted by the pieces that
// open one, and the k-th row's start and stop are written by whichever pieces open and close it.
struct RunPieces {
    int64_t s, e, v, c;
    int64_t pieces;             // 0: the run gives no row
    bool open, close;
};

__device__ __forceinline__ RunPieces run_pieces(const ToIntervalsArgs &a, const int64_t *ends, int64_t i) {
    RunPieces r{a.starts[i], a.starts[i + 1], a.values[i], 0, 0, false, false};
    if (!a.all && r.v == 0) return r;
    const int64_t nc = a.n_contigs;
    r.c = upper_bound(ends, 0, nc + 1, r.s) - 1;                 // ends[c] <= s < ends[c + 1]
    const int64_t c1 = lower_bound(ends, r.c + 1, nc + 1, r.e);   // ends[c1 - 1] < e <= ends[c1]
    r.pieces = c1 - r.c;
    r.open = a.all || i == 0 || ends[r.c] == r.s || a.values[i - 1] == 0;
    r.close = a.all || i == a.n_runs - 1 || (c1 <= nc && ends[c1] == r.e) || a.values[i + 1] == 0;
    return r;
}

__global__ void __launch_bounds__(kScanThreads) runs_to_intervals_kernel(const __grid_constant__ ToIntervalsArgs a) {
    __shared__ ScanSmem sm;
    __shared__ int64_t s_ends[kEndsSmem];
    const int64_t n = a.n_runs, nc = a.n_contigs;
    const bool staged = nc < kEndsSmem;
    if (staged)
        for (int64_t c = threadIdx.x; c <= nc; c += kScanThreads) s_ends[c] = a.ends[c];
    // next_tile's barrier orders the staging before the first search
    const int64_t *ends = staged ? s_ends : a.ends;
    const int64_t n_tiles = (n + kScanTile - 1) / kScanTile;
    for (int64_t tile; (tile = next_tile(a.ws, n_tiles, sm)) >= 0;) {
        const int64_t i0 = tile * kScanTile + (int64_t)threadIdx.x * kScanItems;
        const int64_t i1 = min(i0 + kScanItems, n);
        uint64_t count = 0;
        for (int64_t i = i0; i < i1; ++i) {
            const RunPieces r = run_pieces(a, ends, i);
            if (r.pieces) count += (uint64_t)r.pieces - 1 + r.open;
        }
        uint64_t o = block_exclusive<Sum>(count, tile, a.ws + kWsHeaderWords, sm);
        // the same pieces again (the runs are in L1): keeping eight runs' pieces in registers would spill
        for (int64_t i = i0; i < i1; ++i) {
            const RunPieces r = run_pieces(a, ends, i);
            if (!r.pieces) continue;
            int64_t row = (int64_t)o - !r.open;
            for (int64_t p = 0; p < r.pieces; ++p, ++row) {
                const bool last = p + 1 == r.pieces;
                if (p || r.open) {
                    a.out_contig[row] = (int32_t)(r.c + p);
                    a.out_start[row] = p ? ends[r.c + p] : r.s;
                    if (a.all) a.out_value[row] = r.v;
                }
                if (!last || r.close) a.out_stop[row] = last ? r.e : ends[r.c + p + 1];
            }
            o += (uint64_t)r.pieces - 1 + r.open;
        }
        if (tile == n_tiles - 1 && threadIdx.x == kScanThreads - 1) a.n_out[0] = (int64_t)o;
    }
}

}  // namespace
}  // namespace bnpk

using namespace bnpk;

extern "C" {

int bnpk_interval_events(const int64_t *start, const int64_t *stop, const int32_t *ids, const int64_t *contig_offset,
                         const int64_t *contig_len, size_t n_contigs, int64_t size, size_t n_rows, int64_t *keys,
                         int64_t *g_start, int64_t *g_stop, int64_t *status, void *stream) {
    if (ids && (!contig_offset || !contig_len)) return set_err(BNPK_E_BADARG, "contig ids need contig_offset and contig_len");
    if (!ids && (size < 0 || size >= kMaxPos)) return set_err(BNPK_E_BADARG, "size must be in [0, 2^59)");
    if (n_rows == 0) return 0;
    if (!start || !stop || !status) return set_err(BNPK_E_BADARG, "start, stop and status are required");
    EventArgs a{start, stop, ids, contig_offset, contig_len, (int64_t)n_contigs, size, (int64_t)n_rows,
                keys, g_start, g_stop, status};
    return launch("interval_events_kernel", interval_events_kernel, grid_cap((n_rows + 255) / 256, 8), 256, 0,
                  (cudaStream_t)stream, false, a);
}

int bnpk_pileup_runs(const int64_t *keys, size_t n_keys, int64_t size, int mode, int64_t *run_starts,
                     int64_t *run_values, int64_t *n_runs, void *workspace, size_t workspace_bytes, void *stream) {
    if (mode != BNPK_PILEUP_COUNT && mode != BNPK_PILEUP_ANY) return set_err(BNPK_E_BADARG, "unknown pileup mode");
    if (size < 0 || size >= kMaxPos) return set_err(BNPK_E_BADARG, "size must be in [0, 2^59)");
    if ((n_keys && !keys) || !run_starts || !run_values || !n_runs || !workspace)
        return set_err(BNPK_E_BADARG, "keys, run_starts, run_values, n_runs and workspace are required");
    cudaStream_t st = (cudaStream_t)stream;
    size_t n_tiles;
    if (int rc = scan_workspace(n_keys, 2, workspace, workspace_bytes, st, n_tiles)) return rc;
    return launch("pileup_runs_kernel", pileup_runs_kernel, grid_cap(n_tiles, 4), kScanThreads, 0, st, false,
                  (const int64_t *)keys, (int64_t)n_keys, size, (int)(mode == BNPK_PILEUP_ANY), run_starts, run_values,
                  n_runs, (uint64_t *)workspace);
}

int bnpk_runs_reduce(const int64_t *run_starts, const int64_t *values, size_t n_runs, const int64_t *q_start,
                     const int64_t *q_stop, size_t n_q, int mode, int64_t *out, int64_t *scratch, void *workspace,
                     size_t workspace_bytes, void *stream) {
    if (mode < BNPK_RUNS_MAX || mode > BNPK_RUNS_ANY) return set_err(BNPK_E_BADARG, "unknown reduction");
    if (n_runs < 1 || !run_starts || !values) return set_err(BNPK_E_BADARG, "at least one run is required");
    if (n_q == 0) return 0;
    if (!q_start || !q_stop || !out || !scratch || !workspace)
        return set_err(BNPK_E_BADARG, "q_start, q_stop, out, scratch and workspace are required");
    cudaStream_t st = (cudaStream_t)stream;
    size_t n_tiles;
    if (int rc = scan_workspace(n_q, 1, workspace, workspace_bytes, st, n_tiles)) return rc;
    RunArgs a{run_starts, values, (int64_t)n_runs, q_start, q_stop, (int64_t)n_q, mode,
              scratch, scratch + n_q, scratch + 2 * n_q, out};
    int rc = launch("runs_locate_kernel", runs_locate_kernel, grid_cap((n_q + 255) / 256, 8), 256, 0, st, false, a);
    if (rc) return rc;
    rc = launch("count_scan_kernel", count_scan_kernel, grid_cap(n_tiles, 4), kScanThreads, 0, st, false,
                (const int64_t *)a.count, (int64_t)n_q, a.offs, (uint64_t *)workspace);
    if (rc) return rc;
    // the flat work list is as long as the device says; the grid fills the GPU and strides over it
    return launch("runs_reduce_kernel", runs_reduce_kernel, grid_cap((size_t)-1, 8), 256, 0, st, false, a);
}

int bnpk_runs_extract(const int64_t *run_starts, const int64_t *values, size_t n_runs, const int64_t *q_start,
                      size_t n_q, const int64_t *out_offsets, int64_t *out, void *stream) {
    if (n_runs < 1 || !run_starts || !values) return set_err(BNPK_E_BADARG, "at least one run is required");
    if (n_q == 0) return 0;
    if (!q_start || !out_offsets || !out) return set_err(BNPK_E_BADARG, "q_start, out_offsets and out are required");
    ExtractArgs a{run_starts, values, (int64_t)n_runs, q_start, (int64_t)n_q, out_offsets, out};
    return launch("runs_extract_kernel", runs_extract_kernel, grid_cap((size_t)-1, 8), 256, 0, (cudaStream_t)stream,
                  false, a);
}

int bnpk_interval_merge(const int64_t *start, const int64_t *stop, const uint8_t *same_prev, size_t n_rows,
                        int64_t distance, int64_t *out_rows, int64_t *out_stops, int64_t *n_out, int64_t *status,
                        void *workspace, size_t workspace_bytes, void *stream) {
    if (distance < 0 || distance >= kMaxPos) return set_err(BNPK_E_BADARG, "distance must be in [0, 2^59)");
    if (!n_out) return set_err(BNPK_E_BADARG, "n_out is required");
    cudaStream_t st = (cudaStream_t)stream;
    if (n_rows == 0) {
        BNPK_CUDA(cudaMemsetAsync(n_out, 0, sizeof(int64_t), st));
        return 0;
    }
    if (!start || !stop || !out_rows || !out_stops || !status || !workspace)
        return set_err(BNPK_E_BADARG, "start, stop, out_rows, out_stops, status and workspace are required");
    size_t n_tiles;
    if (int rc = scan_workspace(n_rows, 2, workspace, workspace_bytes, st, n_tiles)) return rc;
    MergeArgs a{start, stop, same_prev, (int64_t)n_rows, distance, out_rows, out_stops, n_out, status,
                (uint64_t *)workspace};
    return launch("interval_merge_kernel", interval_merge_kernel, grid_cap(n_tiles, 4), kScanThreads, 0, st, false, a);
}

int bnpk_rows_equal_prev(const uint8_t *base, size_t base_bytes, const int64_t *starts, const int32_t *lens,
                         size_t n_rows, uint8_t *flag, void *stream) {
    (void)base_bytes;
    if (n_rows == 0) return 0;
    if (!base || !starts || !lens || !flag) return set_err(BNPK_E_BADARG, "base, starts, lens and flag are required");
    return launch("rows_equal_prev_kernel", rows_equal_prev_kernel, grid_cap((n_rows + 255) / 256, 8), 256, 0,
                  (cudaStream_t)stream, false, base, starts, lens, (int64_t)n_rows, flag);
}

int bnpk_runs_combine(const int64_t *a_starts, const int64_t *a_values, size_t n_a, const int64_t *b_starts,
                      const int64_t *b_values, size_t n_b, int op, int64_t *out_starts, int64_t *out_values,
                      int64_t *n_out, void *workspace, size_t workspace_bytes, void *stream) {
    if (op < BNPK_OP_ADD || op > BNPK_OP_GE) return set_err(BNPK_E_BADARG, "unknown track operator");
    if (!a_starts || !b_starts || !out_starts || !n_out || !workspace)
        return set_err(BNPK_E_BADARG, "a_starts, b_starts, out_starts, n_out and workspace are required");
    if ((n_a == 0) != (n_b == 0)) return set_err(BNPK_E_BADARG, "a track without runs is empty: both must be");
    if (n_a && (!a_values || !b_values || !out_values))
        return set_err(BNPK_E_BADARG, "a_values, b_values and out_values are required");
    cudaStream_t st = (cudaStream_t)stream;
    if (n_a == 0) {
        // two tracks of size 0 without runs: no run, and the end of the last run is 0
        BNPK_CUDA(cudaMemsetAsync(n_out, 0, sizeof(int64_t), st));
        BNPK_CUDA(cudaMemsetAsync(out_starts, 0, sizeof(int64_t), st));
        return 0;
    }
    size_t n_tiles;
    if (int rc = scan_workspace(n_a + n_b, 1, workspace, workspace_bytes, st, n_tiles)) return rc;
    CombineArgs a{a_starts, a_values, b_starts, b_values, (int64_t)n_a, (int64_t)n_b, op,
                  out_starts, out_values, n_out, (uint64_t *)workspace};
    return launch("runs_combine_kernel", runs_combine_kernel, grid_cap(n_tiles, 4), kScanThreads, 0, st, false, a);
}

int bnpk_interval_intersect(const int64_t *start, const int64_t *stop, const uint8_t *same_prev, size_t n,
                            int64_t *out_rows, int64_t *out_stops, int64_t *n_out, int64_t *overlap, void *workspace,
                            size_t workspace_bytes, void *stream) {
    if (!n_out) return set_err(BNPK_E_BADARG, "n_out is required");
    if (out_rows && !out_stops) return set_err(BNPK_E_BADARG, "out_rows needs out_stops");
    cudaStream_t st = (cudaStream_t)stream;
    if (n && (!start || !stop || !workspace)) return set_err(BNPK_E_BADARG, "start, stop and workspace are required");
    size_t n_tiles = 0;
    if (n) {
        if (int rc = scan_workspace(n, 1, workspace, workspace_bytes, st, n_tiles)) return rc;
    }
    if (overlap) BNPK_CUDA(cudaMemsetAsync(overlap, 0, sizeof(int64_t), st));
    if (n == 0) {
        BNPK_CUDA(cudaMemsetAsync(n_out, 0, sizeof(int64_t), st));
        return 0;
    }
    IntersectArgs a{start, stop, same_prev, (int64_t)n, out_rows, out_stops, n_out, overlap, (uint64_t *)workspace};
    return launch("interval_intersect_kernel", interval_intersect_kernel, grid_cap(n_tiles, 4), kScanThreads, 0, st,
                  false, a);
}

int bnpk_runs_to_intervals(const int64_t *run_starts, const int64_t *values, size_t n_runs, const int64_t *contig_ends,
                           size_t n_contigs, int mode, int32_t *out_contig, int64_t *out_start, int64_t *out_stop,
                           int64_t *out_value, int64_t *n_out, void *workspace, size_t workspace_bytes, void *stream) {
    if (mode != BNPK_RUNS_TO_NONZERO && mode != BNPK_RUNS_TO_ALL) return set_err(BNPK_E_BADARG, "unknown rows mode");
    if (!n_out) return set_err(BNPK_E_BADARG, "n_out is required");
    cudaStream_t st = (cudaStream_t)stream;
    if (n_runs == 0) {
        BNPK_CUDA(cudaMemsetAsync(n_out, 0, sizeof(int64_t), st));
        return 0;
    }
    if (n_contigs < 1 || n_contigs >= (size_t)INT32_MAX) return set_err(BNPK_E_BADARG, "n_contigs must be in [1, 2^31 - 1)");
    if (!run_starts || !values || !contig_ends || !out_contig || !out_start || !out_stop || !workspace ||
        (mode == BNPK_RUNS_TO_ALL && !out_value))
        return set_err(BNPK_E_BADARG, "run_starts, values, contig_ends, the outputs and workspace are required");
    size_t n_tiles;
    if (int rc = scan_workspace(n_runs, 1, workspace, workspace_bytes, st, n_tiles)) return rc;
    ToIntervalsArgs a{run_starts, values, (int64_t)n_runs, contig_ends, (int64_t)n_contigs,
                      (int)(mode == BNPK_RUNS_TO_ALL), out_contig, out_start, out_stop, out_value, n_out,
                      (uint64_t *)workspace};
    return launch("runs_to_intervals_kernel", runs_to_intervals_kernel, grid_cap(n_tiles, 4), kScanThreads, 0, st,
                  false, a);
}

}  // extern "C"
