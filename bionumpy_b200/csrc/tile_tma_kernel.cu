// tile_tma_kernel.cu -- fused count (K6) into global tables, the chunk staged in shared memory by bulk async
// copies (TMA).  Global tables are bound by L2 atomics: this kernel's 21 row warps per SM keep more of them in flight
// than the warp-specialised kernel's 8 (H100 80 GB HBM3 at 700 W: 14.3 instead of 18.7 ms for 2^20 bins, DESIGN.md).
//
// One persistent CTA per SM; the CTA's kGroups thread groups (256 threads each) are independent tile
// pipelines.  A group owns three 16.5 KiB slots (tile + 512 B
// of halo so that the one row crossing the tile end can finish in it); slots are filled by
// cp.async.bulk and signalled on mbarriers, so no thread ever holds raw bytes in registers across stages.
//
// Per group and iteration i (tiles are handed out in order by an atomic ticket):
//   a. front(P = tile i+1): wait for its bytes; every thread reads its 64 bytes (four conflict-free LDS.128),
//      exact newline mask, warp scan, warp totals -> shared.  One warp finds the first newline of the halo.
//   b. sorted newline list of M = tile i from the masks kept in registers since iteration i-1
//   --- the only group barrier of the iteration ---
//   c. lane 0: publish P's newline count (decoupled look-back), start the bulk copy of tile i+2 into the slot
//      that tile i-1 just left, ask for the next ticket; warp 0 issues P's look-back loads
//   d. one thread per newline validates the entry structure of M; warps 1..7 take the rows in chunks of eight: four
//      threads per row read the row's 16-byte units from the slot, encode + validate them and pass the 2-bit code
//      words round with shuffles; every k-mer is one funnel shift, one mask and one global RED
//   e. warp 0 resolves P's line prefix (its loads had the whole of d to land).  Warp 0 has no rows: it is the group's
//      lowest scheduling priority (the SM arbiter favours high warp ids), so its wait for the predecessors' counts
//      overlaps the other warps' rows instead of following its own.
// A tile's count is public one full iteration before its successor needs it.
#include "tile_common.cuh"

namespace bnpk {
namespace tma {

constexpr int kGroups = 3;
constexpr int kGT = kTileBytes / 64;            // threads per group: one per 64 tile bytes
constexpr int kGW = kGT / 32;
constexpr int kCta = kGroups * kGT;
constexpr int kHalo = 512;
constexpr int kSlot = kTileBytes + kHalo;
constexpr int kSlots = 3;
constexpr int kRowMax = 1024;                   // longer rows go to the deferred (one warp per segment) pass
constexpr int kNlStep = kNlCap - 8;
static_assert(kGT == 256 && kGW == 8, "group geometry");

// per-group control block (32-bit words)
constexpr int kCtlWsum = 0;                     // [kSlots][8] warp totals of the newline counts
constexpr int kCtlCross = 24;                   // [kSlots] first newline of the halo (slot-relative) or kNoCross
constexpr int kCtlTk = 28;                      // [2] ticket broadcast
constexpr int kCtlBase = 32;                    // int64 [2] line index of the tile's first byte
constexpr int kCtlWords = 48;
// shared memory (bytes)
constexpr int kOffSlots = 0;
constexpr int kOffList = kOffSlots + kGroups * kSlots * kSlot;
constexpr int kOffCtl = kOffList + kGroups * 2 * kNlCap * 2;
constexpr int kOffBar = kOffCtl + kGroups * kCtlWords * 4;
constexpr int kOffLut = kOffBar + ((kGroups * kSlots * 8 + 15) & ~15);
constexpr int kFixedBytes = kOffLut + 256;

__device__ __forceinline__ void group_bar(int g) { asm volatile("bar.sync %0, %1;" ::"r"(g + 1), "n"(kGT) : "memory"); }

// HIST: 0 = global int64 table, 2 = global u32 scratch table (the numbering of the other fused-count kernels)
template <int ENC, int HIST>
__global__ void __launch_bounds__(kCta, 1) tile_tma_kernel(const TileArgs a) {
    extern __shared__ __align__(128) uint8_t s_fixed[];
    const int tid = threadIdx.x, g = tid / kGT, gt = tid % kGT, lane = gt & 31, gw = gt >> 5;
    uint8_t *g_slots = s_fixed + kOffSlots + g * (kSlots * kSlot);
    uint16_t *g_list = reinterpret_cast<uint16_t *>(s_fixed + kOffList) + g * (2 * kNlCap);
    uint32_t *g_ctl = reinterpret_cast<uint32_t *>(s_fixed + kOffCtl) + g * kCtlWords;
    int64_t *g_base = reinterpret_cast<int64_t *>(g_ctl + kCtlBase);
    const uint32_t g_bar = smem_addr(s_fixed + kOffBar) + g * (kSlots * 8);
    uint8_t *s_lut = s_fixed + kOffLut;

    const LookbackArrays lb = lookback_arrays(a.ws, a.n_tiles_total);
    const bool cr = a.status[BNPK_ST_CR] != 0;

    if (ENC == BNPK_ENC_LUT && tid < 256) s_lut[tid] = a.lut[tid];
    if (gt == 0) {
#pragma unroll
        for (int s = 0; s < kSlots; ++s) mbar_init(g_bar + 8 * s, 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    const uint64_t hmask = (a.n_bins & (a.n_bins - 1)) == 0 ? a.n_bins - 1 : 0;
    const uint64_t kmask = (1ull << (2 * a.k)) - 1;
    const bool fast = hmask && hmask <= 0x3FFFFFFFull;
    const uint32_t m32x4 = (uint32_t)(hmask & kmask) << 2;       // byte-offset mask into the table
    uint32_t acc_bases = 0, acc_values = 0;                         // per thread: well inside 32 bits for any chunk
    const uint32_t ls = (uint32_t)a.lpe_shift, pm = (1u << ls) - 1u;
    const uint32_t fl = (uint32_t)a.field_line;
    const uint32_t want = (fl - 1u) & pm;
    const int32_t tile_end = (int32_t)a.tile_end;

    ScanLane sl;                                                    // front end: my 64 bytes of the warp's 2 KiB
    sl.init(lane);
    const uint32_t sub = (uint32_t)lane & 3u;
    const int src1 = (lane & ~3) | (int)((sub + 1u) & 3u), src2 = (lane & ~3) | (int)((sub + 2u) & 3u),
              src3 = (lane & ~3) | (int)((sub + 3u) & 3u);

    auto take_ticket = [&]() -> int32_t {
        const unsigned long long t = (unsigned long long)a.tile_begin + atomicAdd((unsigned long long *)(a.ws + kWsTicket), 1ull);
        return (int32_t)min(t, (unsigned long long)0x7FFFFFFF);
    };
    auto staged_len_of = [&](int32_t tile) -> int {
        return (int)min((size_t)kSlot, a.n - (size_t)tile * kTileBytes);
    };
    auto issue_copy = [&](int32_t tile, int slot) {               // one thread
        const size_t byte0 = (size_t)tile * kTileBytes;
        const uint32_t bytes = (uint32_t)staged_len_of(tile) & ~15u;
        const uint32_t bar = g_bar + 8 * slot;
        if (bytes) {
            mbar_expect_tx(bar, bytes);
            bulk_g2s(smem_addr(g_slots + slot * kSlot), a.chunk + byte0, bytes, bar);
        } else {
            mbar_arrive(bar);
        }
    };
    // front end of one tile (every thread of the group)
    auto front = [&](int32_t tile, int slot, uint32_t parity, uint64_t &nl, uint32_t &ex) {
        const uint8_t *sp = g_slots + slot * kSlot;
        const int staged = staged_len_of(tile);
        mbar_wait(g_bar + 8 * slot, parity);
        if (staged & 15) {                                          // the chunk's last bytes: not a multiple of 16
            const int t0 = staged & ~15;
            if (gt < (staged & 15)) g_slots[slot * kSlot + t0 + gt] = a.chunk[(size_t)tile * kTileBytes + t0 + gt];
            group_bar(g);
        }
        nl = sl.mask64(sp + 2048 * gw);
        const int lim = min(staged, kTileBytes) - 64 * gt;          // my bytes inside the tile proper
        if (lim < 64) nl = lim <= 0 ? 0ull : (nl & (~0ull >> (64 - lim)));
        const uint32_t cnt = (uint32_t)__popcll(nl);
        uint32_t inc = cnt;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const uint32_t t = __shfl_up_sync(0xffffffffu, inc, o);
            if (lane >= o) inc += t;
        }
        ex = inc - cnt;
        if (lane == 31) g_ctl[kCtlWsum + 8 * slot + gw] = inc;
        if (gw == 0) {                                              // first newline of the halo: end of the crossing row
            const int valid = min(max(staged - kTileBytes - 16 * lane, 0), 16);
            const uint32_t mm = newline_mask16(lds128(sp + kTileBytes + 16 * lane)) & ((1u << valid) - 1u);
            const unsigned b = __ballot_sync(0xffffffffu, mm != 0);
            const int srcl = b ? __ffs(b) - 1 : 0;
            const uint32_t pos = (uint32_t)(kTileBytes + 16 * lane + __ffs(mm) - 1);
            const uint32_t first = __shfl_sync(0xffffffffu, pos, srcl);
            if (lane == 0) g_ctl[kCtlCross + slot] = b ? first : kNoCross;
        }
    };

    // ---- prologue ---------------------------------------------------------------------------------------
    int32_t tF = 0, t_next = 0;                                     // lane 0 of warp 0 only
    if (gt == 0) {
        const int32_t t0 = take_ticket(), t1 = take_ticket();
        tF = take_ticket();
        g_ctl[kCtlTk + 0] = (uint32_t)t0;
        g_ctl[kCtlTk + 1] = (uint32_t)t1;
        if (t0 < tile_end) issue_copy(t0, 0);
        if (t1 < tile_end) issue_copy(t1, 1);
    }
    group_bar(g);
    int32_t tM = (int32_t)g_ctl[kCtlTk + 0], tP = (int32_t)g_ctl[kCtlTk + 1];
    uint64_t nlM = 0, lbA = kFlagPrefix, lbB = kFlagPrefix;
    uint32_t exM = 0;
    if (tM < tile_end) front(tM, 0, 0u, nlM, exM);
    group_bar(g);                                                   // warp totals of M visible; ticket words free
    if (gw == 0 && tM < tile_end) {
        const uint32_t v = lane < kGW ? g_ctl[kCtlWsum + lane] : 0u;
        const uint32_t cntM = __reduce_add_sync(0xffffffffu, v);
        if (lane == 0) lookback_publish(lb, tM, cntM);
        lookback_issue(lb, tM, lane, lbA, lbB);
        const uint64_t excl = lookback_finish(lb, tM, cntM, lane, lbA, lbB);
        if (lane == 0) g_base[0] = (int64_t)excl;
    }
    int slotM = 0, slotP = 1;
    uint32_t parP = 0;
    uint32_t mb = 0;                                                // iteration parity: list / base / ticket buffers

    while (tM < tile_end) {
        const bool hasP = tP < tile_end;
        const int slotF = slotM == 0 ? 2 : slotM - 1;               // the slot the previous tile just left
        // ---- a. front end of the pending tile ----------------------------------------------------------
        uint64_t nlP = 0;
        uint32_t exP = 0;
        if (hasP) front(tP, slotP, parP, nlP, exP);
        // ---- b. sorted newline list of the main tile (window 0) ----------------------------------------
        const uint8_t *sp = g_slots + slotM * kSlot;
        const size_t byte0 = (size_t)tM * kTileBytes;
        const int staged = staged_len_of(tM);
        uint32_t tile_nl, my_excl;
        {
            const uint32_t v = lane < kGW ? g_ctl[kCtlWsum + 8 * slotM + lane] : 0u;
            tile_nl = __reduce_add_sync(0xffffffffu, v);
            my_excl = exM + __reduce_add_sync(0xffffffffu, lane < gw ? v : 0u);
        }
        uint16_t *list = g_list + mb * kNlCap;
        emit_positions(nlM, my_excl, 64u * (uint32_t)gt, list, 0u);
        if (gt == 0) g_ctl[kCtlTk + mb] = (uint32_t)tF;
        group_bar(g);                                               // ---- the barrier ----
        // ---- c. publish P, refill the free slot, next ticket, P's look-back loads ------------------------
        uint32_t cntP = 0;
        if (gw == 0) {
            if (hasP) {
                const uint32_t v = lane < kGW ? g_ctl[kCtlWsum + 8 * slotP + lane] : 0u;
                cntP = __reduce_add_sync(0xffffffffu, v);
            }
            if (lane == 0) {
                if (hasP) lookback_publish(lb, tP, cntP);
                if (tF < tile_end) {
                    issue_copy(tF, slotF);
                    t_next = take_ticket();
                } else {
                    t_next = tF;
                }
            }
            if (hasP) lookback_issue(lb, tP, lane, lbA, lbB);
        }
        // ---- d. the main tile -------------------------------------------------------------------------
        const int64_t line_base = g_base[mb];
        const uint32_t crossM = g_ctl[kCtlCross + slotM];
        const uint32_t base_phase = (uint32_t)line_base & pm;
        const int64_t q0 = line_base >> ls;                         // entry index of the tile's first line
        const uint32_t jr0 = (want - base_phase) & pm;              // first newline (rel) that precedes a field line
        const int64_t r_first = q0 + ((base_phase + jr0 + 1u) >> ls);
        const int n_rows_tile = (tile_nl > jr0) ? (int)(((tile_nl - 1u - jr0) >> ls) + 1u) : 0;
        const int n_rounds = tile_nl > (uint32_t)kNlCap ? (int)((tile_nl - 8u + kNlStep - 1) / kNlStep) : 1;
        for (int round = 0; round < n_rounds; ++round) {
            const int win_lo = round * kNlStep;
            if (round > 0) {                                        // rare: more than kNlCap lines in one tile
                group_bar(g);
                emit_positions(nlM, my_excl, 64u * (uint32_t)gt, list, (uint32_t)win_lo);
                group_bar(g);
            }
            const int n_in_win = min((int)tile_nl - win_lo, kNlCap);
            const int ev_hi = (round == n_rounds - 1) ? n_in_win : kNlStep;
            // one thread per newline: entry structure (one_line_buffer.py:155-173, fastq_buffer.py:38-45)
            for (int i = gt; i < ev_hi; i += kGT) {
                const uint32_t gi = (uint32_t)(win_lo + i);
                const int p = list[i];
                const uint32_t phase = (base_phase + gi) & pm;
                const bool chk_h = phase == pm, chk_p = a.check_plus && phase == 1u;
                if ((chk_h || chk_p) && byte0 + p + 1 < a.n) {
                    const uint32_t c = sp[p + 1];
                    if (chk_h && c != a.header_char)
                        atomicMin((long long *)&a.status[BNPK_ST_BAD_HEADER_ENTRY], (long long)(q0 + ((base_phase + gi + 1u) >> ls)));
                    if (chk_p && c != '+')
                        atomicMin((long long *)&a.status[BNPK_ST_BAD_PLUS_ENTRY], (long long)(q0 + ((base_phase + gi) >> ls)));
                }
            }
            if (gt == 0 && tile_nl > 0) {                           // last complete entry of the tile
                const uint32_t last = tile_nl - 1u;
                const uint32_t back = (base_phase + last - pm) & pm;
                if (last >= back) {
                    const int li = (int)(last - back) - win_lo;
                    if (li >= 0 && li < ev_hi)
                        atomicMax((unsigned long long *)&a.status[BNPK_ST_N_COMPLETE_BYTES], (unsigned long long)(byte0 + list[li] + 1));
                }
            }
            if (tM == 0 && gt == 0 && round == 0) {
                if (a.n > 0 && sp[0] != a.header_char) atomicMin((long long *)&a.status[BNPK_ST_BAD_HEADER_ENTRY], 0ll);
            }
            // rows whose start newline lies in this window: four threads per row
            const int s_lo = (win_lo > (int)jr0) ? (int)((win_lo - jr0 + pm) >> ls) : 0;
            int s_hi = n_rows_tile;
            if (round != n_rounds - 1) s_hi = min(s_hi, (int)((win_lo + kNlStep - (int)jr0 + (int)pm) >> ls));
            // chunks of 8 rows go round the warps 1..7; warp 0 (look-back, copies, tickets) takes none
            for (int s0 = s_lo + 8 * (gw - 1); gw != 0 && s0 < s_hi; s0 += 8 * (kGW - 1)) {
                const int s = s0 + (lane >> 2);
                bool act = s < s_hi;
                int b0 = 0, e = 0;
                if (act) {
                    const int li = (int)(jr0 + ((uint32_t)s << ls)) - win_lo;
                    b0 = (int)list[li] + 1;
                    if ((uint32_t)(win_lo + li) + 1u < tile_nl) {
                        e = list[li + 1];
                    } else if (crossM != kNoCross) {
                        e = (int)crossM;
                    } else {                                        // not terminated inside the slot
                        if (sub == 0 && byte0 + staged < a.n) defer_row(a, byte0 + b0, (uint64_t)(r_first + s));
                        act = false;                                // (else: unterminated last line, not an entry)
                    }
                    if (act && cr && e > b0 && sp[e - 1] == '\r') e -= 1;
                    if (act && e - b0 > kRowMax) {
                        if (sub == 0) defer_row(a, byte0 + b0, (uint64_t)(r_first + s));
                        act = false;
                    }
                }
                const int L = act ? e - b0 : 0;
                const int npos = max(L - a.k + 1, 0);
                if (act && sub == 0) {
                    acc_bases += (uint32_t)L;
                    acc_values += (uint32_t)npos;
                    if (s == n_rows_tile - 1) {                     // the tile's last counted row (see uncount_kernel)
                        atomicMax((unsigned long long *)&a.status[BNPK_ST_LAST_ROW_START], (unsigned long long)(byte0 + b0) + 1ull);
                        atomicMax((unsigned long long *)&a.status[BNPK_ST_LAST_ROW_INDEX], (unsigned long long)(r_first + s) + 1ull);
                    }
                }
                const int A0 = b0 >> 4, A1 = (e - 1) >> 4;
                const uint32_t o = (uint32_t)b0 & 15u;
                const int my_rounds = L > 0 ? ((A1 - A0 + 1) + 3) >> 2 : 0;
                const int R = __reduce_max_sync(0xffffffffu, my_rounds);
                auto enc = [&](int r) -> uint32_t {
                    const int u = A0 + 4 * r + (int)sub;
                    if (L <= 0 || u > A1) return 0u;
                    const uint4 q = lds128(sp + 16 * u);
                    const int lo = max(b0 - 16 * u, 0), hi = min(e - 16 * u, 16);
                    const uint32_t seq16 = (0xFFFFu >> (16 - hi)) & (0xFFFFu << lo);
                    uint32_t bad;
                    const uint32_t codes = encode_unit<ENC, false>(q, seq16, s_lut, bad);
                    if (bad) report_bad_base<ENC>(a, sp, 16 * u + lo, 16 * u + hi, b0, r_first + s, s_lut);
                    return codes;
                };
                uint32_t c_cur = enc(0);
                for (int r = 0; r < R; ++r) {
                    const uint32_t c_nxt = enc(r + 1);
                    // code words of the next aligned units of my row: lanes of my quad, this round or the next
                    const uint32_t x1 = __shfl_sync(0xffffffffu, c_cur, src1), y1 = __shfl_sync(0xffffffffu, c_nxt, src1);
                    const uint32_t x2 = __shfl_sync(0xffffffffu, c_cur, src2), y2 = __shfl_sync(0xffffffffu, c_nxt, src2);
                    const uint32_t w1 = sub + 1u >= 4u ? y1 : x1, w2 = sub + 2u >= 4u ? y2 : x2;
                    const int left = npos - 16 * (4 * r + (int)sub);       // k-mers that start in my block of 16 bases
                    if (fast) {
                        if (__any_sync(0xffffffffu, left > 0)) {
                            // stream pre-shifted left by two bits: (window & mask) is the table's byte offset
                            const bool z = o == 0u;
                            const uint32_t p0 = z ? 0u : c_cur, p1 = z ? c_cur : w1, p2 = z ? w1 : w2;
                            const uint32_t sh = (2u * o + 30u) & 31u;
                            const uint32_t a0 = __funnelshift_r(p0, p1, sh), a1 = __funnelshift_r(p1, p2, sh);
#pragma unroll
                            for (int t = 0; t < 16; ++t) {
                                const uint32_t v = (t == 0 ? a0 : __funnelshift_r(a0, a1, 2 * t)) & m32x4;
                                if (t < left) {
                                    if constexpr (HIST == 2) atomicAdd(reinterpret_cast<uint32_t *>(reinterpret_cast<char *>(a.hist32) + v), 1u);
                                    else atomicAdd(reinterpret_cast<unsigned long long *>(reinterpret_cast<char *>(a.hist) + 2 * (size_t)v), 1ull);
                                }
                            }
                        }
                    } else {
                        const uint32_t x3 = __shfl_sync(0xffffffffu, c_cur, src3), y3 = __shfl_sync(0xffffffffu, c_nxt, src3);
                        const uint32_t w3 = sub + 3u >= 4u ? y3 : x3;
                        if (left > 0) {
                            const uint32_t sh = 2u * o;
                            const uint32_t a0 = __funnelshift_r(c_cur, w1, sh), a1 = __funnelshift_r(w1, w2, sh),
                                           a2 = __funnelshift_r(w2, w3, sh);
#pragma unroll 4
                            for (int t = 0; t < 16; ++t) {
                                if (t < left) {
                                    const uint32_t lo32 = __funnelshift_r(a0, a1, 2 * t), hi32 = __funnelshift_r(a1, a2, 2 * t);
                                    const uint64_t h = (((uint64_t)hi32 << 32) | lo32) & kmask;
                                    const uint64_t b = hmask ? (h & hmask) : (h % a.n_bins);
                                    if constexpr (HIST == 2) atomicAdd(a.hist32 + b, 1u);
                                    else atomicAdd(a.hist + b, 1ull);
                                }
                            }
                        }
                    }
                    c_cur = c_nxt;
                }
            }
        }
        if (tM == (int32_t)(a.n_tiles_total - 1) && gt == 0) a.status[BNPK_ST_N_LINES] = line_base + tile_nl;
        // ---- e. the pending tile's line prefix; rotate ---------------------------------------------------
        if (gw == 0 && hasP) {
            const uint64_t excl = lookback_finish(lb, tP, cntP, lane, lbA, lbB);
            if (lane == 0) g_base[mb ^ 1u] = (int64_t)excl;
        }
        tM = tP; nlM = nlP; exM = exP;
        tP = (int32_t)g_ctl[kCtlTk + mb];
        if (gt == 0) tF = t_next;
        slotM = slotP;
        slotP = slotP == kSlots - 1 ? 0 : slotP + 1;
        if (slotP == 0) parP ^= 1u;
        mb ^= 1u;
    }

    // ---- flush ---------------------------------------------------------------------------------------------
    const uint64_t sum_bases = warp_sum_u64(acc_bases), sum_values = warp_sum_u64(acc_values);
    if (lane == 0) {
        if (sum_bases) atomicAdd((unsigned long long *)&a.status[BNPK_ST_N_BASES], sum_bases);
        if (sum_values) atomicAdd((unsigned long long *)&a.status[BNPK_ST_N_VALUES], sum_values);
    }
}

template <int ENC, int HIST>
static int launch_t(const TileArgs &a, cudaStream_t st) {
    auto kern = tile_tma_kernel<ENC, HIST>;
    BNPK_DYN_SMEM(kern, kFixedBytes);
    const int64_t n_tiles = a.tile_end - a.tile_begin;
    if (n_tiles <= 0) return 0;
    return launch("tile_tma_kernel", kern, grid_cap((size_t)(n_tiles + kGroups - 1) / kGroups, 1), kCta, kFixedBytes, st,
                  true, a);
}

template <int ENC>
static int launch_enc(const TileArgs &a, cudaStream_t st) {
    return a.hist32 ? launch_t<ENC, 2>(a, st) : launch_t<ENC, 0>(a, st);
}

}  // namespace tma

// k-mer counts into global tables; bulk copies need a 16-byte-aligned chunk, tile indices stay in 31 bits
bool tma_count_eligible(const TileArgs &a, bool smem_hist) {
    if (a.window != 0 || smem_hist) return false;
    if ((reinterpret_cast<uintptr_t>(a.chunk) & 15) != 0) return false;
    return a.tile_end <= 0x7FFFFFF0ll && a.n >= 16;
}

int launch_tma_count(const TileArgs &a, int enc_mode, cudaStream_t st) {
    return with_enc(enc_mode, [&](auto enc) { return tma::launch_enc<decltype(enc)::value>(a, st); });
}

}  // namespace bnpk
