// bam_kernels.cu -- BAM records on the device (BamBuffer._find_starts / BamBufferExtractor, io/bam.py:18-331;
// split_cigar / count_reference_length, alignments/cigar.py:8-24).
//
// Records are chained by their block_size words, so the split is a speculative segmented walk (DESIGN §3 K15):
//   bam_speculate_kernel : a warp per segment tests 32 candidate offsets at a time (ballot) for a plausible record
//                          chain, and one lane walks from the first one to the first record start at or past the
//                          segment's end.
//   bam_resolve_kernel   : one warp confirms the segments in order from offset 0.  A window of 32 segments whose
//                          speculative starts are each the exit of the segment before is taken whole; any other window
//                          is resolved segment by segment, and a segment whose speculative start is not the confirmed
//                          entry is walked again from that entry.  The running record count gives each segment's
//                          output offset.
//   bam_starts_kernel    : one thread per segment walks its confirmed records again and writes their starts.
// bam_fields_kernel reads the fixed 36 bytes of one record per thread; the unpack kernels spread their output bytes
// over the threads and find each thread's first row by binary search of the row offsets.
#include "bnpk_host.h"

namespace bnpk {

namespace {

constexpr int kBamFixed = 36;     // block_size word + the 32 fixed bytes
constexpr int kChainDepth = 4;    // records after a candidate that must pass too, while they lie in the chunk
constexpr int kSpecWarps = 4;
constexpr int kRecTail = -1;      // check_record: the record does not end inside the chunk
constexpr int kRecOk = 0;
constexpr int kSeqItems = 16;
constexpr int kCigarItems = 4;

// workspace rows (int64[7][n_seg])
enum { kSpecStart, kSpecExit, kSpecCount, kSpecState, kConfEntry, kConfCount, kConfOffset, kWsRows };

__device__ __forceinline__ uint32_t ld_u16(const uint8_t *p) { return (uint32_t)__ldg(p) | (uint32_t)__ldg(p + 1) << 8; }
__device__ __forceinline__ uint32_t ld_u32(const uint8_t *p) { return ld_u16(p) | ld_u16(p + 2) << 16; }

// kRecOk (a complete record that passes the header check; `next` is the offset after it), kRecTail, or the
// BNPK_BAM_BAD_* of the first check the bytes inside the chunk fail
__device__ int check_record(const uint8_t *c, int64_t n, int64_t p, int n_ref, int64_t &next) {
    if (p + 4 > n) return kRecTail;
    const int64_t bs = ld_u32(c + p);
    next = p + 4 + bs;
    if (bs < 32) return BNPK_BAM_BAD_BLOCK_SIZE;
    if (p + kBamFixed > n) return kRecTail;
    const int32_t ref = (int32_t)ld_u32(c + p + 4), next_ref = (int32_t)ld_u32(c + p + 24);
    if (ref < -1 || ref >= n_ref || next_ref < -1 || next_ref >= n_ref) return BNPK_BAM_BAD_REF_ID;
    const int64_t l_name = __ldg(c + p + 12), n_cigar = ld_u16(c + p + 16), l_seq = (int32_t)ld_u32(c + p + 20);
    if (l_name == 0) return BNPK_BAM_BAD_NAME;
    if (l_seq < 0 || 32 + l_name + 4 * n_cigar + (l_seq + 1) / 2 + l_seq > bs) return BNPK_BAM_BAD_SIZES;
    if (next > n) return kRecTail;
    if (__ldg(c + p + kBamFixed + l_name - 1) != 0) return BNPK_BAM_BAD_NAME;
    return kRecOk;
}

// a candidate record start: a complete record that passes the check, followed by kChainDepth more that pass while
// they lie in the chunk.  The candidate itself must be complete: a random block_size is mostly huge, and bytes near 0
// pass the header check, so an incomplete first record says nothing.
__device__ bool plausible(const uint8_t *c, int64_t n, int64_t p, int n_ref) {
    for (int d = 0; d <= kChainDepth; ++d) {
        int64_t next = p;
        const int r = check_record(c, n, p, n_ref, next);
        if (r != kRecOk) return r == kRecTail && d > 0;
        p = next;
    }
    return true;
}

// walks the records from p while p < end; count += the records passed; returns 0 (reached end), kRecTail or the
// BNPK_BAM_BAD_* of the record at p
__device__ int walk(const uint8_t *c, int64_t n, int n_ref, int64_t &p, int64_t end, int64_t &count) {
    while (p < end) {
        int64_t next = p;
        const int r = check_record(c, n, p, n_ref, next);
        if (r != kRecOk) return r;
        p = next;
        ++count;
    }
    return 0;
}

struct SplitArgs {
    const uint8_t *chunk;
    int64_t n, seg, n_seg;
    int n_ref;
    int64_t *ws;
    int64_t *starts;
    int64_t *status;
};

__global__ void __launch_bounds__(kSpecWarps * 32) bam_speculate_kernel(const __grid_constant__ SplitArgs a) {
    const int lane = threadIdx.x & 31;
    const int64_t s = (int64_t)blockIdx.x * kSpecWarps + (threadIdx.x >> 5);
    if (s >= a.n_seg) return;
    const int64_t lo = s * a.seg, hi = min(lo + a.seg, a.n);
    int64_t start = s == 0 ? 0 : -1;
    for (int64_t o = lo; s != 0 && o < hi; o += 32) {
        const int64_t q = o + lane;
        const unsigned hit = __ballot_sync(0xffffffffu, q < hi && plausible(a.chunk, a.n, q, a.n_ref));
        if (hit) {
            start = o + __ffs(hit) - 1;
            break;
        }
    }
    if (lane) return;
    int64_t p = start, count = 0;
    const int state = start < 0 ? 0 : walk(a.chunk, a.n, a.n_ref, p, hi, count);
    int64_t *ws = a.ws;
    ws[kSpecStart * a.n_seg + s] = start;
    ws[kSpecExit * a.n_seg + s] = p;
    ws[kSpecCount * a.n_seg + s] = count;
    ws[kSpecState * a.n_seg + s] = state;
}

__global__ void __launch_bounds__(32) bam_resolve_kernel(const __grid_constant__ SplitArgs a) {
    const int lane = threadIdx.x;
    const int64_t ns = a.n_seg;
    const int64_t *spec = a.ws;
    int64_t *conf = a.ws + kConfEntry * ns;
    int64_t cur = 0, total = 0, redo = 0;
    int state = 0;
    for (int64_t s0 = 0; s0 < ns && state == 0; s0 += 32) {
        const int64_t s = s0 + lane;
        const bool in = s < ns;
        const int64_t start = in ? spec[kSpecStart * ns + s] : -1, exit = in ? spec[kSpecExit * ns + s] : 0;
        const int64_t count = in ? spec[kSpecCount * ns + s] : 0;
        const int64_t sstate = in ? spec[kSpecState * ns + s] : 0;
        const int64_t prev_exit = __shfl_up_sync(0xffffffffu, exit, 1);
        const int64_t entry = lane ? prev_exit : cur;
        if (__all_sync(0xffffffffu, !in || (start == entry && sstate == 0))) {
            // every segment of the window stands
            int64_t inc = count;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const int64_t t = __shfl_up_sync(0xffffffffu, inc, o);
                if (lane >= o) inc += t;
            }
            if (in) {
                conf[s] = start;
                conf[ns + s] = count;
                conf[2 * ns + s] = total + inc - count;
            }
            const int last = (int)(ns - 1 - s0 < 31 ? ns - 1 - s0 : 31);
            total += __shfl_sync(0xffffffffu, inc, last);
            cur = __shfl_sync(0xffffffffu, exit, last);
            continue;
        }
        if (lane == 0) {
            for (int64_t t = s0; t < min(s0 + 32, ns) && state == 0; ++t) {
                const int64_t seg_end = min((t + 1) * a.seg, a.n);
                int64_t e = -1, k = 0;
                if (cur < seg_end) {
                    e = cur;
                    if (spec[kSpecStart * ns + t] == cur) {
                        k = spec[kSpecCount * ns + t];
                        cur = spec[kSpecExit * ns + t];
                        state = (int)spec[kSpecState * ns + t];
                    } else {
                        ++redo;
                        state = walk(a.chunk, a.n, a.n_ref, cur, seg_end, k);
                    }
                }
                conf[t] = e;
                conf[ns + t] = k;
                conf[2 * ns + t] = total;
                total += k;
            }
        }
        cur = __shfl_sync(0xffffffffu, cur, 0);
        total = __shfl_sync(0xffffffffu, total, 0);
        state = __shfl_sync(0xffffffffu, state, 0);
    }
    if (lane == 0) {
        a.status[BNPK_ST_N_RECORDS] = total;
        a.status[BNPK_ST_N_COMPLETE_BYTES] = cur;
        a.status[BNPK_ST_N_VALUES] = redo;
        if (state > 0) a.status[BNPK_ST_BAD_BASE] = total << 8 | state;
    }
}

__global__ void __launch_bounds__(256) bam_starts_kernel(const __grid_constant__ SplitArgs a) {
    const int64_t ns = a.n_seg;
    const int64_t *conf = a.ws + kConfEntry * ns;
    for (int64_t s = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; s < ns; s += (int64_t)gridDim.x * blockDim.x) {
        int64_t p = conf[s], o = conf[2 * ns + s];
        const int64_t end = o + conf[ns + s];
        for (; o < end; ++o) {
            a.starts[o] = p;
            p += 4 + (int64_t)ld_u32(a.chunk + p);
        }
    }
}

__global__ void __launch_bounds__(256) bam_fields_kernel(const uint8_t *c, const int64_t *starts, int64_t max_records,
                                                         int64_t *f, int64_t *status) {
    const int64_t n = min(max_records, (int64_t)status[BNPK_ST_N_RECORDS]);
    for (int64_t r = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; r < n; r += (int64_t)gridDim.x * blockDim.x) {
        const int64_t p = starts[r];
        const int64_t l_name = __ldg(c + p + 12), n_cigar = ld_u16(c + p + 16), l_seq = (int32_t)ld_u32(c + p + 20);
        const int64_t name = p + kBamFixed, cigar = name + l_name, seq = cigar + 4 * n_cigar;
        int64_t ref_len = 0;
        bool bad_op = false;
        for (int64_t j = 0; j < n_cigar; ++j) {
            const uint32_t w = ld_u32(c + cigar + 4 * j), op = w & 15;
            bad_op |= op > 8;
            // M (0), D (2), N (3), = (7) and X (8) consume the reference
            if ((0x18du >> op) & 1) ref_len += w >> 4;
        }
        if (bad_op) atomicMin((long long *)&status[BNPK_ST_BAD_BASE], (long long)(r << 8 | BNPK_BAM_BAD_CIGAR_OP));
        f[BNPK_BAM_F_REF_ID * max_records + r] = (int32_t)ld_u32(c + p + 4);
        f[BNPK_BAM_F_POS * max_records + r] = (int32_t)ld_u32(c + p + 8);
        f[BNPK_BAM_F_MAPQ * max_records + r] = __ldg(c + p + 13);
        f[BNPK_BAM_F_FLAG * max_records + r] = ld_u16(c + p + 18);
        f[BNPK_BAM_F_NAME_START * max_records + r] = name;
        f[BNPK_BAM_F_NAME_LEN * max_records + r] = l_name - 1;
        f[BNPK_BAM_F_CIGAR_START * max_records + r] = cigar;
        f[BNPK_BAM_F_N_CIGAR * max_records + r] = n_cigar;
        f[BNPK_BAM_F_SEQ_START * max_records + r] = seq;
        f[BNPK_BAM_F_L_SEQ * max_records + r] = l_seq;
        f[BNPK_BAM_F_QUAL_START * max_records + r] = seq + (l_seq + 1) / 2;
        f[BNPK_BAM_F_REF_LEN * max_records + r] = ref_len;
    }
}

// the row that holds output item j: the last r with offsets[r] <= j (rows of length 0 are skipped)
__device__ __forceinline__ int64_t row_of(const int64_t *offsets, int64_t n_rows, int64_t j) {
    int64_t lo = 0, hi = n_rows;          // offsets[lo] <= j < offsets[hi]
    while (hi - lo > 1) {
        const int64_t mid = (lo + hi) >> 1;
        if (offsets[mid] <= j) lo = mid; else hi = mid;
    }
    return lo;
}

__global__ void __launch_bounds__(256) bam_sequence_kernel(const uint8_t *c, const int64_t *seq_start,
                                                           const int64_t *offsets, int64_t n_rows, uint8_t *out) {
    const int64_t total = offsets[n_rows];
    for (int64_t j0 = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) * kSeqItems; j0 < total;
         j0 += (int64_t)gridDim.x * blockDim.x * kSeqItems) {
        int64_t r = row_of(offsets, n_rows, j0);
        const int64_t j1 = min(j0 + kSeqItems, total);
        for (int64_t j = j0; j < j1; ++j) {
            while (offsets[r + 1] <= j) ++r;
            const int64_t i = j - offsets[r];
            const uint8_t b = __ldg(c + seq_start[r] + (i >> 1));
            out[j] = (i & 1) ? (b & 15) : (b >> 4);
        }
    }
}

__global__ void __launch_bounds__(256) bam_cigar_kernel(const uint8_t *c, const int64_t *cigar_start,
                                                        const int64_t *offsets, int64_t n_rows, uint8_t *op,
                                                        int64_t *length) {
    const int64_t total = offsets[n_rows];
    for (int64_t j0 = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) * kCigarItems; j0 < total;
         j0 += (int64_t)gridDim.x * blockDim.x * kCigarItems) {
        int64_t r = row_of(offsets, n_rows, j0);
        const int64_t j1 = min(j0 + kCigarItems, total);
        for (int64_t j = j0; j < j1; ++j) {
            while (offsets[r + 1] <= j) ++r;
            const uint32_t w = ld_u32(c + cigar_start[r] + 4 * (j - offsets[r]));
            op[j] = (uint8_t)(w & 15);
            length[j] = w >> 4;
        }
    }
}

}  // namespace

}  // namespace bnpk

using namespace bnpk;

extern "C" {

int bnpk_bam_split(const uint8_t *chunk, size_t n, int n_ref, size_t segment_bytes, int64_t *starts, size_t max_starts,
                   int64_t *status, int64_t *workspace, size_t workspace_words, void *stream) {
    if (n_ref < 0 || segment_bytes < 64) return set_err(BNPK_E_BADARG, "n_ref >= 0 and segment_bytes >= 64");
    if (!status) return set_err(BNPK_E_BADARG, "status is required");
    const int64_t n_seg = (int64_t)((n + segment_bytes - 1) / segment_bytes);
    if (n == 0) return 0;
    if (!chunk || !starts || !workspace) return set_err(BNPK_E_BADARG, "chunk, starts and workspace are required");
    if (max_starts < n / kBamFixed) return set_err(BNPK_E_BADARG, "max_starts must be at least n / 36");
    if (workspace_words < (size_t)(kWsRows * n_seg)) return set_err(BNPK_E_WORKSPACE, "workspace too small");
    const cudaStream_t st = (cudaStream_t)stream;
    const SplitArgs a{chunk, (int64_t)n, (int64_t)segment_bytes, n_seg, n_ref, workspace, starts, status};
    // segments after a stop are never confirmed: they keep no records
    BNPK_CUDA(cudaMemsetAsync(workspace + kConfEntry * n_seg, 0, 3 * n_seg * sizeof(int64_t), st));
    int rc =launch("bam_speculate_kernel", bam_speculate_kernel, (unsigned)((n_seg + kSpecWarps - 1) / kSpecWarps),
                    kSpecWarps * 32, 0, st, false, a);
    if (rc) return rc;
    if ((rc = launch("bam_resolve_kernel", bam_resolve_kernel, 1, 32, 0, st, false, a))) return rc;
    return launch("bam_starts_kernel", bam_starts_kernel, grid_cap((n_seg + 255) / 256, 8), 256, 0, st, false, a);
}

int bnpk_bam_fields(const uint8_t *chunk, size_t /* n: the records lie inside it */, const int64_t *starts,
                    size_t max_records, int64_t *fields, int64_t *status, void *stream) {
    if (max_records == 0) return 0;
    if (!chunk || !starts || !fields || !status) return set_err(BNPK_E_BADARG, "chunk, starts, fields and status are required");
    return launch("bam_fields_kernel", bam_fields_kernel, grid_cap((max_records + 255) / 256, 8), 256, 0,
                  (cudaStream_t)stream, false, chunk, starts, (int64_t)max_records, fields, status);
}

int bnpk_bam_sequence(const uint8_t *chunk, size_t /* n */, const int64_t *seq_start, const int64_t *offsets,
                      size_t n_rows, uint8_t *out, void *stream) {
    if (n_rows == 0) return 0;
    if (!chunk || !seq_start || !offsets || !out) return set_err(BNPK_E_BADARG, "chunk, seq_start, offsets and out are required");
    return launch("bam_sequence_kernel", bam_sequence_kernel, grid_cap((size_t)-1, 8), 256, 0, (cudaStream_t)stream,
                  false, chunk, seq_start, offsets, (int64_t)n_rows, out);
}

int bnpk_bam_cigar(const uint8_t *chunk, size_t /* n */, const int64_t *cigar_start, const int64_t *offsets,
                   size_t n_rows, uint8_t *op, int64_t *length, void *stream) {
    if (n_rows == 0) return 0;
    if (!chunk || !cigar_start || !offsets || !op || !length)
        return set_err(BNPK_E_BADARG, "chunk, cigar_start, offsets, op and length are required");
    return launch("bam_cigar_kernel", bam_cigar_kernel, grid_cap((size_t)-1, 8), 256, 0, (cudaStream_t)stream, false,
                  chunk, cigar_start, offsets, (int64_t)n_rows, op, length);
}

}  // extern "C"
