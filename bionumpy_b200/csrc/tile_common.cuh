// tile_common.cuh -- pieces shared by the tile kernels (tile_kernels.cu: split + register-staged count;
// tile_ws_kernel.cu: the warp-specialised counts; tile_tma_kernel.cu: the count into global tables): launch
// arguments, the rare-path helpers, the bulk-copy / mbarrier wrappers, the newline list of a staged tile and the
// two-level decoupled look-back over the tile newline counts.
#pragma once
#include "bnpk_host.h"

namespace bnpk {

struct TileArgs {
    const uint8_t *chunk;
    size_t n;
    int64_t tile_begin, tile_end;  // tiles handled by this launch
    int lpe, lpe_shift, field_line, start_offset;
    uint32_t header_char;
    int check_plus;
    int64_t *status;
    uint64_t *ws;                  // header | tile_state[] | deferred[]
    int64_t n_tiles_total;
    uint64_t *deferred;            // long-row list (start, entry) pairs
    size_t deferred_cap;
    // split
    int64_t *starts;
    int32_t *lens;
    size_t max_rows;
    // count
    const uint8_t *lut;
    int k, window;                 // window = 0: k-mers; else minimizers over `window` bases
    uint64_t n_bins;
    unsigned long long *hist;
    uint32_t *hist32;              // optional 32-bit scratch table in the workspace (large global tables), else null
};

// first bad byte of a row some encode_unit flagged -> the BAD_BASE status word
template <int ENC>
__device__ __forceinline__ void report_bad_base(const TileArgs &a, const uint8_t *bytes, int p0, int p1, int b0, int64_t entry,
                                                const uint8_t *s_lut) {
    const int64_t v = first_bad_base<ENC>(bytes, p0, p1, b0, entry, s_lut);
    if (v != INT64_MAX) report_fault(a.status, v);
}

// A row the kernel cannot finish (no newline inside the staged bytes, or too long for its row walk): (first byte, entry)
// goes to the deferred list that count_fixups_impl counts afterwards.
__device__ __forceinline__ void defer_row(const TileArgs &a, uint64_t start, uint64_t r) {
    const unsigned long long d = atomicAdd((unsigned long long *)(a.ws + kWsDeferred), 1ull);
    if (d < a.deferred_cap) {
        a.deferred[2 * d] = start;
        a.deferred[2 * d + 1] = r;
    } else {
        a.status[BNPK_ST_OVERFLOW] = 1;
    }
}

// ---- shared-memory staging by bulk copies (tile_ws_kernel.cu, tile_tma_kernel.cu) ------------------------------
__device__ __forceinline__ uint32_t smem_addr(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
// try_wait with a suspend-time hint; sleeping between the tests (nanosleep 64) costs more in wake-up latency than the
// polling costs in issue slots, so the loop polls.
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "WAIT_%=:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1, %2;\n"
        "@p bra DONE_%=;\n"
        "bra WAIT_%=;\n"
        "DONE_%=:\n"
        "}\n" ::"r"(bar), "r"(parity), "r"(20000u)
        : "memory");
}
__device__ __forceinline__ void bulk_g2s(uint32_t dst, const void *src, uint32_t bytes, uint32_t bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst),
                 "l"(src), "r"(bytes), "r"(bar)
                 : "memory");
}
__device__ __forceinline__ uint4 lds128(const uint8_t *p) { return *reinterpret_cast<const uint4 *>(p); }
// one count into the CTA-private table (32-bit shared address)
__device__ __forceinline__ void hist_inc(uint32_t addr) { asm volatile("red.shared.add.u32 [%0], 1;" ::"r"(addr) : "memory"); }
// ptxas never predicates ATOMS (it branches around it), so a masked count adds 0 or 1 instead
__device__ __forceinline__ void hist_add_val(uint32_t addr, uint32_t val) { asm volatile("red.shared.add.u32 [%0], %1;" ::"r"(addr), "r"(val) : "memory"); }
// The 16 k-mers of one block of a lane's row into the CTA-private table (table bins a power of two).  K-mer t is the
// field at bit 2t of (cur, nxt), the row's 2-bit codes from the block's first base on; shifted two bits less,
// (window & mask) is its byte offset.  FULL (the block is full in every row of the warp): the offset is
// (window & mask) | dummy, one LOP3 -- mask 0 and dummy = the spare word behind the table for a lane without a row.
// Otherwise k-mers t >= left (left = the lane's k-mers that start in this block) count into the spare word `dummy`:
// a select per k-mer, no branch.
template <bool FULL>
__device__ __forceinline__ void count_block16(uint32_t hist_sa, uint32_t cur, uint32_t nxt, uint32_t mask, uint32_t dummy, int left) {
#pragma unroll
    for (int t = 0; t < 16; ++t) {
        const uint32_t win = t == 0 ? cur << 2 : __funnelshift_r(cur, nxt, 2 * t - 2);
        hist_inc(hist_sa + (FULL ? (win & mask) | dummy : t < left ? win & mask : dummy));
    }
}

// ---- the sorted newline list of a tile (emit_positions: every tile kernel; ScanLane: the kernels that stage tiles in
// shared-memory slots) ---------------------------------------------------------------------------------------------
constexpr int kNlCap = 1024;                    // newline positions of one tile kept in shared memory
constexpr uint32_t kNoCross = 0xFFFFFFFFu;      // no newline in the halo

// Conflict-free read of a lane's 64 bytes (LDS.128 j fetches unit (j + lane/2) & 3) -> exact 64-bit newline mask.
struct ScanLane {
    uint32_t off[4], sel_lo, sel_hi;
    __device__ __forceinline__ void init(int lane) {
        const uint32_t rot = ((uint32_t)lane >> 1) & 3u;
#pragma unroll
        for (int j = 0; j < 4; ++j) off[j] = 64u * (uint32_t)lane + 16u * (((uint32_t)j + rot) & 3u);
        // halfword h of the byte-order mask comes from load (h - rot) & 3; PRMT byte pair of load jj in
        // (A = m0|m1<<16, B = m2|m3<<16) is 0x10 + 0x22*jj
        sel_lo = (0x10u + 0x22u * ((0u - rot) & 3u)) | ((0x10u + 0x22u * ((1u - rot) & 3u)) << 8);
        sel_hi = (0x10u + 0x22u * ((2u - rot) & 3u)) | ((0x10u + 0x22u * ((3u - rot) & 3u)) << 8);
    }
    // p = base of the warp's 2 KiB piece
    __device__ __forceinline__ uint64_t mask64(const uint8_t *p) const {
        uint32_t m[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) m[j] = newline_mask16(lds128(p + off[j]));
        const uint32_t A = m[1] * 65536u + m[0], B = m[3] * 65536u + m[2];
        return ((uint64_t)prmt(A, B, sel_hi) << 32) | prmt(A, B, sel_lo);
    }
};

// write the positions of the set bits of m (tile-relative base `pos`) at list[li - wb ...] when inside the window
__device__ __forceinline__ void emit_positions(uint64_t m, uint32_t li, uint32_t pos, uint16_t *list, uint32_t wb) {
    uint32_t lo = (uint32_t)m, hi = (uint32_t)(m >> 32);
    while (lo) {
        const int bit = __ffs((int)lo) - 1;
        lo &= lo - 1;
        if (li - wb < (uint32_t)kNlCap) list[li - wb] = (uint16_t)(pos + bit);
        ++li;
    }
    while (hi) {
        const int bit = __ffs((int)hi) - 1;
        hi &= hi - 1;
        if (li - wb < (uint32_t)kNlCap) list[li - wb] = (uint16_t)(pos + 32 + bit);
        ++li;
    }
}

// ---- two-level look-back state in the workspace ------------------------------------------------
//   tile_state[t]  : flag|value, AGG = newlines of tile t, PREFIX = newlines of tiles 0..t
//   block_cnt[b]   : atomic (count << 56 | sum) over the 32 tiles of block b
//   block_state[b] : flag|value, AGG = newlines of the whole block, PREFIX = newlines of tiles 0..32b+31
// A tile resolves its exclusive prefix from <= 31 tile entries of its own block plus <= 32 block
// entries: two loads per lane, issued one pipeline stage before they are needed.
struct LookbackArrays {
    uint64_t *tile_state, *block_cnt, *block_state;
};
__device__ __forceinline__ LookbackArrays lookback_arrays(uint64_t *ws, int64_t n_tiles_total) {
    LookbackArrays l;
    l.tile_state = ws + kWsHeaderWords;
    const int64_t nb = (n_tiles_total >> 5) + 2;
    l.block_cnt = l.tile_state + n_tiles_total + 1;
    l.block_state = l.block_cnt + nb;
    return l;
}
__device__ __forceinline__ void lookback_publish(const LookbackArrays &l, int64_t tile, uint64_t agg) {
    st_relaxed(l.tile_state + tile, (tile == 0 ? kFlagPrefix : kFlagAgg) | agg);
    const int64_t b = tile >> 5;
    const unsigned long long old = atomicAdd((unsigned long long *)(l.block_cnt + b), (1ull << 56) | agg);
    if ((old >> 56) == 31ull)
        atomicMax((unsigned long long *)(l.block_state + b), kFlagAgg | ((old & ((1ull << 56) - 1)) + agg));
}
__device__ __forceinline__ void lookback_issue(const LookbackArrays &l, int64_t tile, int lane, uint64_t &lbA, uint64_t &lbB) {
    const int i = (int)(tile & 31);
    const int64_t b = tile >> 5;
    lbA = (lane < i) ? ld_relaxed(l.tile_state + tile - 1 - lane) : kFlagPrefix;
    lbB = (b - 1 - lane >= 0) ? ld_relaxed(l.block_state + (b - 1 - lane)) : kFlagPrefix;
}
// Warp-wide.  Returns the exclusive prefix of `tile` and publishes its inclusive prefix.
__device__ __forceinline__ uint64_t lookback_finish(const LookbackArrays &l, int64_t tile, uint64_t agg, int lane,
                                                    uint64_t lbA, uint64_t lbB) {
    const int i = (int)(tile & 31);
    int64_t b = tile >> 5;
    uint64_t excl = 0;
    bool have = false;
    // ---- my own block: tiles 32b .. tile-1 (lane 0 = tile-1).  Wait (a short loop: the waiting warp shares its
    // issue slots with the warps it waits for) until every earlier tile of the block has published something.
    {
        const bool valid = lane < i;
        while (__any_sync(0xffffffffu, valid && (lbA >> 62) == 0))
            if (valid && (lbA >> 62) == 0) lbA = ld_relaxed(l.tile_state + tile - 1 - lane);
        const unsigned pref = __ballot_sync(0xffffffffu, valid && (lbA >> 62) == 2);
        const unsigned upto = pref ? ((pref & (0u - pref)) << 1) - 1u : 0xffffffffu;     // lanes 0..first prefix
        const uint64_t v = (valid && ((1u << lane) & upto)) ? (lbA & kValueMask) : 0;
        excl = warp_sum_u64(v);
        have = pref != 0;
    }
    // ---- whole blocks before mine (lane 0 = block b-1)
    int64_t bb = b;
    while (!have) {
        const unsigned pref = __ballot_sync(0xffffffffu, (lbB >> 62) == 2);
        const unsigned zero = __ballot_sync(0xffffffffu, (lbB >> 62) == 0);
        const unsigned upto = pref ? ((pref & (0u - pref)) << 1) - 1u : 0xffffffffu;
        if (zero & upto) {
            lbB = (bb - 1 - lane >= 0) ? ld_relaxed(l.block_state + (bb - 1 - lane)) : kFlagPrefix;
            continue;
        }
        const uint64_t v = ((1u << lane) & upto) ? (lbB & kValueMask) : 0;
        excl += warp_sum_u64(v);
        if (pref) break;
        bb -= 32;                                            // more than 32 blocks back (cold start only)
        lbB = (bb - 1 - lane >= 0) ? ld_relaxed(l.block_state + (bb - 1 - lane)) : kFlagPrefix;
    }
    if (lane == 0) {
        const uint64_t incl = (excl + agg) & kValueMask;
        st_relaxed(l.tile_state + tile, kFlagPrefix | incl);
        if (i == 31) atomicMax((unsigned long long *)(l.block_state + b), kFlagPrefix | incl);
    }
    return excl;
}

// The fused-count kernels besides the register-staged tile_kernel, which takes every call none of them is eligible for.
// smem_hist = the table is counted in a CTA-private shared-memory table (use_smem_hist).
// warp-specialised, minimizers (tile_ws_kernel.cu): windows of up to 12 k-mers, CTA-private table of up to 2^14 bins,
// 16-byte-aligned chunk
bool wsm_count_eligible(const TileArgs &a, bool smem_hist);
int launch_wsm_count(const TileArgs &a, int enc_mode, cudaStream_t st);
// warp-specialised, k-mers: CTA-private table of up to 2^14 bins, aligned chunk
bool ws_count_eligible(const TileArgs &a, bool smem_hist);
int launch_ws_count(const TileArgs &a, int enc_mode, cudaStream_t st);
// shared-memory-staged (tile_tma_kernel.cu), k-mers: global table, aligned chunk
bool tma_count_eligible(const TileArgs &a, bool smem_hist);
int launch_tma_count(const TileArgs &a, int enc_mode, cudaStream_t st);
constexpr int64_t kScratch32MaxBins = 1ll << 24;   // 64 MiB of u32 counters at the end of the workspace

}  // namespace bnpk
