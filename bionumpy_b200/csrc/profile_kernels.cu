// profile_kernels.cu -- column sums of equal-length windows of a run-length track (K18): the meta-profile
// track[windows].mean(axis=0) around TSSs or peak summits, without writing a value per position.
//
// column_sum_kernel<V>: one CTA per (block of BNPK_COLUMN_BLOCK_ROWS rows, tile of kColTile columns), grid-strided.
//   Each thread first locates one row of the block: the span of positions the tile covers in that row (reversed rows
//   read it back to front) and the runs that overlap it, found by binary search in the global run starts.  The span is
//   kColTile positions at most and runs are non-empty, so at most kColTile runs overlap it.  Rows are then staged
//   kStageRows at a time, one warp per row copying its runs into shared memory, and every thread adds, for its own
//   column, the value of the run that holds its position (a binary search over the staged starts) into a register,
//   in row order from +0.0.  The block's sums go to partial[b * width + j].
// column_fold_kernel<V>: one thread per column adds the block partials in block order from +0.0; the loads of
//   kFoldUnroll blocks are issued before their adds.  No atomics: a float64 sum has the same bits on every call.
#include "bnpk_host.h"

namespace bnpk {

namespace {

constexpr int kColTile = 256;              // columns of a CTA, one per thread
constexpr int kStageRows = 8;              // rows staged per pair of barriers, one warp each
constexpr int kFoldUnroll = 16;            // block partials loaded ahead of their adds in the fold
constexpr int kFoldThreads = 32;           // one warp per fold CTA: the few columns spread over many SMs
static_assert(BNPK_COLUMN_BLOCK_ROWS % kStageRows == 0, "a block is whole stages");
static_assert(kStageRows * 32 <= kColTile, "one warp per staged row");

template <typename V>
struct ColumnArgs {
    const int64_t *starts;       // int64[R + 1]
    const V *values;             // V[R]
    int64_t n_runs;
    const int64_t *q_start;
    const uint8_t *reverse;      // may be null: no row reversed
    int64_t n_q, width;
    V *out, *partial;
    int64_t n_blocks, n_tiles;
};

// int64 sums wrap (added as unsigned); float64 sums round once per add, never contracted
__device__ __forceinline__ int64_t add_value(int64_t a, int64_t b) { return (int64_t)((uint64_t)a + (uint64_t)b); }
__device__ __forceinline__ double add_value(double a, double b) { return __dadd_rn(a, b); }

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

template <typename V>
__global__ void __launch_bounds__(kColTile) column_sum_kernel(const __grid_constant__ ColumnArgs<V> a) {
    __shared__ int64_t s_lo[BNPK_COLUMN_BLOCK_ROWS];       // the first position of the tile's span in each row
    __shared__ int64_t s_run[BNPK_COLUMN_BLOCK_ROWS];      // the run that holds it
    __shared__ int32_t s_cnt[BNPK_COLUMN_BLOCK_ROWS];      // the runs that overlap the span
    __shared__ uint8_t s_rev[BNPK_COLUMN_BLOCK_ROWS];
    __shared__ int64_t s_starts[kStageRows][kColTile + 1];
    __shared__ V s_values[kStageRows][kColTile];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int64_t n_items = a.n_blocks * a.n_tiles;
    for (int64_t item = blockIdx.x; item < n_items; item += gridDim.x) {
        const int64_t b = item / a.n_tiles, j0 = (item % a.n_tiles) * kColTile;
        const int len = (int)min((int64_t)kColTile, a.width - j0);
        const int64_t q0 = b * BNPK_COLUMN_BLOCK_ROWS;
        const int rows = (int)min((int64_t)BNPK_COLUMN_BLOCK_ROWS, a.n_q - q0);
        for (int r = tid; r < rows; r += kColTile) {
            const int64_t q = q0 + r;
            const bool rev = a.reverse && a.reverse[q];
            const int64_t lo = a.q_start[q] + (rev ? a.width - j0 - len : j0);
            const int64_t r0 = first_above(a.starts, 1, a.n_runs, lo) - 1;
            const int64_t r1 = first_at_least(a.starts, r0 + 1, min(r0 + len, a.n_runs), lo + len);
            s_lo[r] = lo;
            s_run[r] = r0;
            s_cnt[r] = (int32_t)(r1 - r0);
            s_rev[r] = rev;
        }
        __syncthreads();
        V acc = V(0);
        for (int s0 = 0; s0 < rows; s0 += kStageRows) {
            const int n_stage = min(kStageRows, rows - s0);
            if (warp < n_stage) {
                const int64_t r0 = s_run[s0 + warp];
                const int cnt = s_cnt[s0 + warp];
                for (int i = lane; i <= cnt; i += 32) {
                    s_starts[warp][i] = a.starts[r0 + i];
                    if (i < cnt) s_values[warp][i] = a.values[r0 + i];
                }
            }
            __syncthreads();
            if (tid < len) {
                for (int w = 0; w < n_stage; ++w) {
                    const int r = s0 + w;
                    const int64_t p = s_lo[r] + (s_rev[r] ? len - 1 - tid : tid);
                    // the last staged run whose start is <= p
                    int k = 0, n = s_cnt[r];
                    while (n > 1) {
                        const int half = n >> 1;
                        k = s_starts[w][k + half] <= p ? k + half : k;
                        n -= half;
                    }
                    acc = add_value(acc, s_values[w][k]);
                }
            }
            __syncthreads();
        }
        if (tid < len) a.partial[b * a.width + j0 + tid] = acc;
    }
}

template <typename V>
__global__ void __launch_bounds__(kFoldThreads) column_fold_kernel(const __grid_constant__ ColumnArgs<V> a) {
    for (int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; j < a.width; j += (int64_t)gridDim.x * blockDim.x) {
        V acc = V(0);
        int64_t b = 0;
        for (; b + kFoldUnroll <= a.n_blocks; b += kFoldUnroll) {
            V v[kFoldUnroll];
#pragma unroll
            for (int u = 0; u < kFoldUnroll; ++u) v[u] = a.partial[(b + u) * a.width + j];
#pragma unroll
            for (int u = 0; u < kFoldUnroll; ++u) acc = add_value(acc, v[u]);
        }
        for (; b < a.n_blocks; ++b) acc = add_value(acc, a.partial[b * a.width + j]);
        a.out[j] = acc;
    }
}

template <typename V>
int column_sum(const int64_t *run_starts, const V *values, size_t n_runs, const int64_t *q_start,
               const uint8_t *reverse, size_t n_q, int64_t width, V *out, V *partial, void *stream) {
    if (width < 0 || width >= ((int64_t)1 << 31)) return set_err(BNPK_E_BADARG, "width must be in [0, 2^31)");
    if (n_runs < 1 || !run_starts || !values)
        return set_err(BNPK_E_BADARG, "run_starts and values of at least one run are required");
    if (width == 0) return 0;
    if (!out) return set_err(BNPK_E_BADARG, "out is required");
    if (n_q && (!q_start || !partial)) return set_err(BNPK_E_BADARG, "q_start and partial are required");
    cudaStream_t st = (cudaStream_t)stream;
    if (n_q == 0) {
        BNPK_CUDA(cudaMemsetAsync(out, 0, (size_t)width * sizeof(V), st));
        return 0;
    }
    const int64_t n_blocks = ((int64_t)n_q + BNPK_COLUMN_BLOCK_ROWS - 1) / BNPK_COLUMN_BLOCK_ROWS;
    const int64_t n_tiles = (width + kColTile - 1) / kColTile;
    const ColumnArgs<V> a{run_starts, values, (int64_t)n_runs, q_start, reverse, (int64_t)n_q, width,
                          out, partial, n_blocks, n_tiles};
    int rc = launch("column_sum_kernel", column_sum_kernel<V>, grid_cap((size_t)(n_blocks * n_tiles), 4), kColTile,
                    0, st, false, a);
    if (rc) return rc;
    return launch("column_fold_kernel", column_fold_kernel<V>, grid_cap((size_t)(width + kFoldThreads - 1) /
                  kFoldThreads, 32), kFoldThreads, 0, st, false, a);
}

}  // namespace
}  // namespace bnpk

extern "C" {

int bnpk_runs_column_sum(const int64_t *run_starts, const int64_t *values, size_t n_runs, const int64_t *q_start,
                         const uint8_t *reverse, size_t n_q, int64_t width, int64_t *out, int64_t *partial,
                         void *stream) {
    return bnpk::column_sum(run_starts, values, n_runs, q_start, reverse, n_q, width, out, partial, stream);
}

int bnpk_track_f64_column_sum(const int64_t *run_starts, const double *values, size_t n_runs, const int64_t *q_start,
                              const uint8_t *reverse, size_t n_q, int64_t width, double *out, double *partial,
                              void *stream) {
    return bnpk::column_sum(run_starts, values, n_runs, q_start, reverse, n_q, width, out, partial, stream);
}

}  // extern "C"
