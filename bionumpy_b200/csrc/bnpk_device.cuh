// bnpk_device.cuh -- shared device helpers for the sm_90a k-mer hot path.
//
// Every kernel that reads sequence bytes classifies them here, one 16-byte unit at a time (see DESIGN.md):
//   newline_mask16 : bit i = "byte i is '\n'"
//   encode_unit    : 2 bits per byte (byte j of the unit at bits 2j) -> a contiguous 2-bit stream, and which bytes are
//                    outside the alphabet of the encoding
//   first_bad_base : the same alphabets one byte at a time, for the rare rescan of a row that holds a bad byte
// A k-mer starting at byte b is the 2k-bit field at bit 2b of the packed stream (first base in the lowest bits), which
// is exactly the reference hash sum_j code[i+j]*4^j (sequence/kmers.py:105-126).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <type_traits>
#include "../../include/bnpk.h"

namespace bnpk {

constexpr int kTileBytes = 16384;          // bytes owned by one tile
constexpr int kHaloBytes = 2048;           // extra bytes staged so in-tile rows can finish
constexpr int kStagedUnits = (kTileBytes + kHaloBytes) / 16; // 1152
constexpr int kSmemMaxBins = 32768;        // u32 bins that fit next to the tile staging

constexpr uint64_t kFlagAgg = 1ull << 62;
constexpr uint64_t kFlagPrefix = 2ull << 62;
constexpr uint64_t kValueMask = (1ull << 62) - 1;

// workspace header (uint64 words)
constexpr int kWsTicket = 0;        // per-launch tile ticket
constexpr int kWsDeferred = 1;      // number of deferred (long) rows
constexpr int kWsCarry = 2;         // newlines in all tiles of the earlier launches (slices) of this chunk
constexpr int kWsRedo = 3;          // ranges the warp-specialised count counted twice (first line phase guessed wrong)
// Deferred rows of one 16 KiB tile the warp-specialised count can produce: rows longer than its 1024-byte row walk
// start more than 1024 bytes apart (<= 16), plus the tile's last row when it ends beyond the slot (1)
constexpr int kWsDeferPerTile = 17;
constexpr int kWsHeaderWords = 16;

__device__ __forceinline__ uint64_t ld_relaxed(const uint64_t *p) {
    uint64_t v;
    asm volatile("ld.relaxed.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void st_relaxed(uint64_t *p, uint64_t v) {
    asm volatile("st.relaxed.gpu.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
// streaming 16-byte load: read-only path, do not keep in L1
__device__ __forceinline__ uint4 ld_stream(const uint4 *p) {
    uint4 r;
    asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
                 : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p));
    return r;
}
// 16 bytes from an arbitrary address, as two aligned 16-byte loads and a funnel shift (both loads touch only the
// aligned blocks that hold bytes of [p, p + 16), so they stay inside the allocation)
__device__ __forceinline__ void load16(const uint8_t *p, uint32_t (&o)[4]) {
    const uintptr_t addr = reinterpret_cast<uintptr_t>(p);
    const uint4 *q = reinterpret_cast<const uint4 *>(addr & ~(uintptr_t)15);
    const int s = (int)(addr & 15);
    const uint4 lo = __ldg(q);
    if (s == 0) {
        o[0] = lo.x; o[1] = lo.y; o[2] = lo.z; o[3] = lo.w;
        return;
    }
    const uint4 hi = __ldg(q + 1);
    const uint32_t w[8] = {lo.x, lo.y, lo.z, lo.w, hi.x, hi.y, hi.z, hi.w};
    const int k = s >> 2, sh = (s & 3) * 8;
    uint32_t t[5];
#pragma unroll
    for (int j = 0; j < 5; ++j) {
        const uint32_t c0 = w[j], c1 = j + 1 < 8 ? w[j + 1] : 0u, c2 = j + 2 < 8 ? w[j + 2] : 0u,
                       c3 = j + 3 < 8 ? w[j + 3] : 0u;
        t[j] = k == 0 ? c0 : k == 1 ? c1 : k == 2 ? c2 : c3;
    }
#pragma unroll
    for (int j = 0; j < 4; ++j) o[j] = __funnelshift_r(t[j], t[j + 1], sh);
}

__device__ __forceinline__ uint64_t warp_sum_u64(uint64_t v) {
#pragma unroll
    for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// ---------------------------------------------------------------------------------------------
// Single-pass scans: tiles of kScanTile items, handed out in increasing order by a ticket and chained by a decoupled
// look-back.  A scan's workspace is kWsHeaderWords header words (the ticket) and one look-back state per tile,
// zeroed before the launch (scan_workspace in bnpk_host.h).
//
// An operator is a type with `static uint64_t combine(uint64_t before, uint64_t after)`, associative and with
// identity 0, on values of the 62-bit field of a look-back state.
// ---------------------------------------------------------------------------------------------
constexpr int kScanThreads = 256;
constexpr int kScanItems = 8;
constexpr int kScanTile = kScanThreads * kScanItems;
constexpr int kScanWarps = kScanThreads / 32;

struct Sum {
    __device__ __forceinline__ static uint64_t combine(uint64_t before, uint64_t after) { return before + after; }
};

struct ScanSmem {
    uint64_t warp[kScanWarps];
    uint64_t base;
    int64_t tile;
};

// The block's next tile, or -1 once the tiles [0, n_tiles) are all handed out.  Every thread of the block calls it,
// and the loop body must pass a __syncthreads() before the next call (block_exclusive does).
__device__ __forceinline__ int64_t next_tile(uint64_t *ws, int64_t n_tiles, ScanSmem &sm) {
    if (threadIdx.x == 0) sm.tile = (int64_t)atomicAdd((unsigned long long *)(ws + kWsTicket), 1ull);
    __syncthreads();
    const int64_t tile = sm.tile;
    return tile < n_tiles ? tile : -1;
}

// The words of the 32 lanes combined, a higher lane before a lower one, in every lane.
template <class Op>
__device__ __forceinline__ uint64_t warp_combine_down(uint64_t v, int lane) {
    if constexpr (std::is_same<Op, Sum>::value) {
        return warp_sum_u64(v);                             // a sum does not depend on the order
    } else {
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const uint64_t t = __shfl_down_sync(0xffffffffu, v, o);
            if (lane + o < 32) v = Op::combine(t, v);
        }
        return __shfl_sync(0xffffffffu, v, 0);
    }
}

// Decoupled look-back.  Called by one full warp.  Publishes this tile's aggregate, walks back over predecessors until
// an inclusive prefix is found, publishes the tile's inclusive prefix and returns the exclusive one.  Tiles are handed
// out in increasing order by the ticket, so every predecessor is already running (or done).  The walk keeps
// kLookbackDepth windows of 32 predecessors in flight per round trip; they are combined from the newest to the oldest.
constexpr int kLookbackDepth = 4;
template <class Op>
__device__ __forceinline__ uint64_t lookback(uint64_t *state, int64_t tile, uint64_t aggregate, int lane) {
    if (tile == 0) {
        if (lane == 0) st_relaxed(state, kFlagPrefix | aggregate);
        return 0;
    }
    if (lane == 0) st_relaxed(state + tile, kFlagAgg | aggregate);
    uint64_t excl = 0;
    int64_t idx = tile - 1;
    while (true) {
        uint64_t s[kLookbackDepth];
        bool pending;
        do {
            pending = false;
#pragma unroll
            for (int d = 0; d < kLookbackDepth; ++d) {
                const int64_t j = idx - 32 * d - lane;
                s[d] = (j >= 0) ? ld_relaxed(state + j) : kFlagPrefix;
            }
            // only entries up to the first inclusive prefix matter
            bool need = true;
#pragma unroll
            for (int d = 0; d < kLookbackDepth; ++d) {
                const unsigned zero = __ballot_sync(0xffffffffu, (s[d] >> 62) == 0);
                const unsigned pref = __ballot_sync(0xffffffffu, (s[d] >> 62) == 2);
                if (need) {
                    // a not-yet-published entry before the first prefix of this window?
                    const unsigned before = pref ? ((pref & (0u - pref)) - 1u) : 0xffffffffu;   // lanes closer than the first prefix
                    if (zero & before) pending = true;
                    if (pref) need = false;
                }
            }
        } while (pending);
        bool done = false;
#pragma unroll
        for (int d = 0; d < kLookbackDepth; ++d) {
            if (!done) {
                const unsigned pmask = __ballot_sync(0xffffffffu, (s[d] >> 62) == 2);
                uint64_t v = s[d] & kValueMask;
                if (pmask) {
                    const int first = __ffs(pmask) - 1;
                    if (lane > first) v = 0;
                    done = true;
                }
                excl = Op::combine(warp_combine_down<Op>(v, lane), excl);
            }
        }
        if (done) break;
        idx -= 32 * kLookbackDepth;
    }
    if (lane == 0) st_relaxed(state + tile, kFlagPrefix | (Op::combine(excl, aggregate) & kValueMask));
    return excl;
}

// The exclusive scan of one value per thread over the whole input: the block's scan, made global by look-back over
// `state` (one word per tile).  Returns this thread's global exclusive prefix.  Every thread of the block calls it.
template <class Op>
__device__ __forceinline__ uint64_t block_exclusive(uint64_t v, int64_t tile, uint64_t *state, ScanSmem &sm) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    uint64_t inc = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const uint64_t t = __shfl_up_sync(0xffffffffu, inc, o);
        if (lane >= o) inc = Op::combine(t, inc);
    }
    if (lane == 31) sm.warp[warp] = inc;
    __syncthreads();
    if (warp == 0) {
        uint64_t winc = lane < kScanWarps ? sm.warp[lane] : 0;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const uint64_t t = __shfl_up_sync(0xffffffffu, winc, o);
            if (lane >= o) winc = Op::combine(t, winc);
        }
        const uint64_t total = __shfl_sync(0xffffffffu, winc, kScanWarps - 1);
        const uint64_t wex = __shfl_up_sync(0xffffffffu, winc, 1);
        if (lane < kScanWarps) sm.warp[lane] = lane ? wex : 0;
        const uint64_t excl = lookback<Op>(state, tile, total & kValueMask, lane);
        if (lane == 0) sm.base = excl;
    }
    __syncthreads();
    // an exclusive prefix is the inclusive one of the lane before: an operator need not have an inverse
    const uint64_t lex = __shfl_up_sync(0xffffffffu, inc, 1);
    const uint64_t r = Op::combine(Op::combine(sm.base, sm.warp[warp]), lane ? lex : 0);
    __syncthreads();                                        // sm is free again
    return r;
}

// offs[i] = size_of(0) + ... + size_of(i - 1) for i in [0, n], so offs[n] is the total, in one pass over a
// one-scan workspace.  size_of(i) >= 0 is called once for every i < n.  Every thread of the block calls it.
template <class F>
__device__ __forceinline__ void exclusive_offsets(int64_t n, int64_t *offs, uint64_t *ws, F size_of) {
    __shared__ ScanSmem sm;
    const int64_t n_tiles = (n + kScanTile - 1) / kScanTile;
    for (int64_t tile; (tile = next_tile(ws, n_tiles, sm)) >= 0;) {
        const int64_t i0 = tile * kScanTile + (int64_t)threadIdx.x * kScanItems;
        uint64_t v[kScanItems];
        uint64_t sum = 0;
#pragma unroll
        for (int j = 0; j < kScanItems; ++j) {
            v[j] = i0 + j < n ? size_of(i0 + j) : 0;
            sum += v[j];
        }
        uint64_t o = block_exclusive<Sum>(sum, tile, ws + kWsHeaderWords, sm);
#pragma unroll
        for (int j = 0; j < kScanItems; ++j) {
            if (i0 + j < n) offs[i0 + j] = (int64_t)o;
            o += v[j];
        }
        if (tile == n_tiles - 1 && threadIdx.x == kScanThreads - 1) offs[n] = (int64_t)o;
    }
}

// ---------------------------------------------------------------------------------------------
// byte classes of a 16-byte unit: the one statement of the alphabets, used by every kernel
// ---------------------------------------------------------------------------------------------
// Integer pipes of an SM sub-partition (tools/micro/pipe_bench.cu): LOP3/SHF/PRMT/IADD3 (ALU pipe) and IMAD /
// IDP.4A (FMA pipe) each issue one warp instruction every two cycles, any mix of the two 0.65 per cycle; POPC one
// every 8 cycles, ffs (BREV + FLO) one every 16.  This path is all integer work: instruction count sets the time.

// PRMT without the selector clean-up __byte_perm adds (all selectors used here are in range)
__device__ __forceinline__ uint32_t prmt(uint32_t lo, uint32_t hi, uint32_t sel) {
    uint32_t d;
    asm("prmt.b32 %0, %1, %2, %3;" : "=r"(d) : "r"(lo), "r"(hi), "r"(sel));
    return d;
}
// bit 7 of every byte that equals '\n' (bit 7 of the pattern is clear, so the last term can use w itself)
__device__ __forceinline__ uint32_t newline_msb(uint32_t w) {
    uint32_t x;                                                     // (w ^ 0x0A..) & 0x7F.. as ONE LOP3
    asm("lop3.b32 %0, %1, 0x0A0A0A0A, 0x7F7F7F7F, 0x28;" : "=r"(x) : "r"(w));
    const uint32_t s = x + 0x7F7F7F7Fu;
    return ~(s | w) & 0x80808080u;
}

// exact '\n' flags of a 16-byte unit, bit i = byte i: the flag bytes are 0x80 or 0, one IDP.4A per word weighs
// them into place (4 instructions per word, two of them on the FMA pipe)
__device__ __forceinline__ uint32_t newline_mask16(const uint4 q) {
    uint32_t lo = __dp4a(newline_msb(q.x), 0x08040201u, 0u);
    lo = __dp4a(newline_msb(q.y), 0x80402010u, lo);                // 128 * (flags of bytes 0..7)
    uint32_t hi = __dp4a(newline_msb(q.z), 0x08040201u, 0u);
    hi = __dp4a(newline_msb(q.w), 0x80402010u, hi);                // 128 * (flags of bytes 8..15)
    return (lo >> 7) | (hi << 1);
}

// 16-byte unit -> 32 bits of 2-bit codes; `bad` != 0 iff a byte of the unit (WHOLE) or a byte selected by seq16
// (!WHOLE) is outside the alphabet (exact).  !WHOLE: `bad` is the 16-bit mask of those bytes, bit i = byte i.
// ASCII alphabets: bits 1-2 of a letter are a Gray code of its index (A 00, C 01, G 11, T 10).  Per word: one LOP3
// isolates them, one IMAD packs the four fields into the top byte, one IMAD lines them up as PRMT selector nibbles,
// PRMT looks the expected lower-case letter up, LOP3 compares it with the case-folded input; per unit: three PRMT
// gather the packed bytes and (ACGT only) two ops turn Gray into binary for all sixteen bases at once.
template <int ENC, bool WHOLE>
__device__ __forceinline__ uint32_t encode_unit(const uint4 q, uint32_t seq16, const uint8_t *s_lut, uint32_t &bad) {
    const uint32_t w[4] = {q.x, q.y, q.z, q.w};
    if constexpr (ENC == BNPK_ENC_ASCII_ACGT || ENC == BNPK_ENC_ASCII_ACTG || ENC == BNPK_ENC_CODES) {
        uint32_t dif[4], pk[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            if constexpr (ENC == BNPK_ENC_CODES) {
                pk[j] = (w[j] & 0x03030303u) * 0x01041040u;
                dif[j] = w[j] & 0xFCFCFCFCu;
            } else {
                const uint32_t g2 = w[j] & 0x06060606u;
                pk[j] = g2 * 0x00820820u;                           // top byte = the four 2-bit fields
                const uint32_t sel = prmt(g2 * 0x110u, 0u, 0x4431u);   // nibbles = 2 * field: 0 a, 2 c, 4 t, 6 g
                dif[j] = prmt(0x00630061u, 0x00670074u, sel) ^ (w[j] | 0x20202020u);
            }
        }
        uint32_t codes = prmt(prmt(pk[0], pk[1], 0x0073), prmt(pk[2], pk[3], 0x0073), 0x5410);
        if constexpr (ENC == BNPK_ENC_ASCII_ACGT) codes ^= (codes >> 1) & 0x55555555u;
        if constexpr (WHOLE) {
            bad = dif[0] | dif[1] | dif[2] | dif[3];
        } else {
            // byte != 0 flags (bit 7 of every byte), weighed into a 16-bit mask like the newline flags
            uint32_t nz[4];
#pragma unroll
            for (int j = 0; j < 4; ++j) nz[j] = (((dif[j] & 0x7F7F7F7Fu) + 0x7F7F7F7Fu) | dif[j]) & 0x80808080u;
            const uint32_t lo = __dp4a(nz[1], 0x80402010u, __dp4a(nz[0], 0x08040201u, 0u));
            const uint32_t hi = __dp4a(nz[3], 0x80402010u, __dp4a(nz[2], 0x08040201u, 0u));
            bad = ((lo >> 7) | (hi << 1)) & seq16;
        }
        return codes;
    } else {
        uint32_t codes = 0;
        bad = 0;
#pragma unroll
        for (int b = 0; b < 16; ++b) {
            const uint32_t code = s_lut[(w[b >> 2] >> (8 * (b & 3))) & 0xFFu];
            codes |= (code & 3u) << (2 * b);
            bad |= ((code >= 4u) ? 1u : 0u) << b;
        }
        if constexpr (!WHOLE) bad &= seq16;
        return codes;
    }
}

// The same alphabets one byte at a time, for the rare rescan of a row some encode_unit flagged: the first byte of
// bytes[p0, p1) outside the alphabet, as (entry << 32 | offset from the row's first byte b0) for the BAD_BASE status
// word (a minimum); INT64_MAX if there is none.
template <int ENC>
__device__ __forceinline__ long long first_bad_base(const uint8_t *bytes, int p0, int p1, int b0, int64_t entry, const uint8_t *s_lut) {
    for (int p = p0; p < p1; ++p) {
        const uint32_t c = bytes[p];
        bool okb;
        if (ENC == BNPK_ENC_CODES) okb = c < 4;
        else if (ENC == BNPK_ENC_LUT) okb = s_lut[c] < 4;
        else { const uint32_t uu = c | 0x20u; okb = (uu == 'a' || uu == 'c' || uu == 'g' || uu == 't'); }
        if (!okb) return (long long)((entry << 32) | (int64_t)(p - b0));
    }
    return INT64_MAX;
}

// load a 16-byte unit that may stick out of [0, n): out-of-range bytes read as 0
__device__ __forceinline__ uint4 load_unit_guarded(const uint8_t *base, size_t n, int64_t unit_byte0) {
    if (unit_byte0 >= 0 && (size_t)unit_byte0 + 16 <= n && ((reinterpret_cast<uintptr_t>(base) + unit_byte0) & 15) == 0)
        return ld_stream(reinterpret_cast<const uint4 *>(base + unit_byte0));
    uint32_t w[4] = {0, 0, 0, 0};
#pragma unroll
    for (int b = 0; b < 16; ++b) {
        const int64_t p = unit_byte0 + b;
        if (p >= 0 && (size_t)p < n) w[b >> 2] |= (uint32_t)base[p] << (8 * (b & 3));
    }
    return make_uint4(w[0], w[1], w[2], w[3]);
}

// length of the line starting at global byte `start` (distance to the next '\n'); -1 if the data
// ends first.  Warp-wide.
__device__ __forceinline__ int64_t warp_line_len(const uint8_t *base, size_t n, int64_t start, int lane) {
    const int off = (int)((reinterpret_cast<uintptr_t>(base) + start) & 15);
    int64_t u0 = start - off;
    bool first = true;
    while (u0 < (int64_t)n) {
        const int64_t ub = u0 + 16 * (int64_t)lane;
        uint32_t m = 0;
        if (ub < (int64_t)n) {
            m = newline_mask16(load_unit_guarded(base, n, ub));
            if (first && lane == 0) m &= 0xFFFFu << off;
        }
        const unsigned b = __ballot_sync(0xffffffffu, m != 0);
        if (b) {
            const int src = __ffs(b) - 1;
            const int64_t pos = ub + __ffs(m) - 1;
            return __shfl_sync(0xffffffffu, pos, src) - start;
        }
        first = false;
        u0 += 512;
    }
    return -1;
}

// ---------------------------------------------------------------------------------------------
// packed-stream readers
// ---------------------------------------------------------------------------------------------
// low 32 bits of the 2-bit stream starting at byte `b` (codes[] is the unit array, 32-bit words)
__device__ __forceinline__ uint32_t stream_lo32(const uint32_t *codes, uint32_t b) {
    const uint32_t bit = 2u * b;
    const uint32_t idx = bit >> 5, sh = bit & 31u;
    return __funnelshift_r(codes[idx], codes[idx + 1], sh);
}
// 64 bits of the stream starting at byte `b`
__device__ __forceinline__ uint64_t stream_64(const uint32_t *codes, uint32_t b) {
    const uint32_t bit = 2u * b;
    const uint32_t idx = bit >> 5, sh = bit & 31u;
    const uint32_t w0 = codes[idx], w1 = codes[idx + 1], w2 = codes[idx + 2];
    return ((uint64_t)__funnelshift_r(w1, w2, sh) << 32) | __funnelshift_r(w0, w1, sh);
}

// sliding minimum over `w` consecutive lanes (w <= 32): lane l gets min(v[l .. l+w-1]);
// only lanes l <= 32-w hold a complete window.
__device__ __forceinline__ uint64_t warp_sliding_min(uint64_t v, int w) {
    int span = 1;
    while (span * 2 <= w) {
        const uint64_t o = __shfl_down_sync(0xffffffffu, v, span);
        v = o < v ? o : v;
        span *= 2;
    }
    const int rest = w - span;
    if (rest) {
        const uint64_t o = __shfl_down_sync(0xffffffffu, v, rest);
        v = o < v ? o : v;
    }
    return v;
}

// min(h, hash of the reverse complement of the k-mer): bases reversed (bit reversal + swap inside each pair) and
// complemented.  cx = the complement as an XOR on every 2-bit code (ACGT order: 3 -> all ones, ACTG order: 2).
__device__ __forceinline__ uint64_t canonical_hash(uint64_t h, int k, uint64_t cx) {
    uint64_t x = __brevll(h ^ cx);
    x = ((x & 0x5555555555555555ull) << 1) | ((x >> 1) & 0x5555555555555555ull);
    x >>= (64 - 2 * k);
    return x < h ? x : h;
}

// 64-bit mixer (Steele, Lea, Flood: SplitMix64's output function after one increment): the synthetic reads' generator and
// the home slot of a key in the k-mer table
__device__ __forceinline__ uint64_t splitmix64(uint64_t x) {
    uint64_t z = x + 0x9E3779B97F4A7C15ull;
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    return z ^ (z >> 31);
}

// ---------------------------------------------------------------------------------------------
// Exact k-mer table: open addressing with linear probing, structure of arrays in global memory.
// keys[slot] == kTableEmpty marks a free slot; a k-mer hash (k <= 31) is below 2^62, so it never equals -1.
// The home slot mixes the key: a raw hash's low bits are its first bases, far from uniform on real genomes.
//
// Why a plain relaxed load of keys[] is enough (no lock, no second pass):
//   * a key slot is written at most once, by the CAS that moves it from EMPTY to a key, and never changes afterwards.
//     So a load that returns a key returns the slot's final value: comparing it with ours is decided for good.
//   * a load that returns EMPTY may be stale (another thread's CAS has landed since).  We then CAS EMPTY -> key; the
//     CAS is atomic at L2 and returns the slot's true value: EMPTY (we claimed the slot), our key (someone else
//     inserted the same k-mer first) or another key (the slot is taken: probe on).  Stale EMPTY is resolved there.
//   * two threads inserting the same k-mer both probe the same sequence from the same home slot, and every slot before
//     the one that holds it is already occupied by another key for good, so they cannot end up in different slots.
//   * counts are only ever incremented with atomicAdd after the slot holds the key; nothing reads them while inserts
//     run (results and rehash are later kernels on the same stream).
// ---------------------------------------------------------------------------------------------
constexpr unsigned long long kTableEmpty = ~0ull;

struct KmerTable {
    unsigned long long *keys;    // int64[capacity], kTableEmpty = free
    unsigned long long *counts;  // int64[capacity]
    uint64_t mask;               // capacity - 1 (capacity a power of two)
    unsigned long long *n_used;  // slots claimed (device counter, aggregated per warp by the callers)
};

__device__ __forceinline__ uint64_t table_home(uint64_t key, uint64_t mask) { return splitmix64(key) & mask; }

// add `count` to `key`'s slot.  Returns 1 if this call claimed a free slot, 0 otherwise; probing every slot without
// finding room drops the key and sets status[BNPK_ST_TABLE_FULL].
__device__ __forceinline__ uint32_t table_insert(const KmerTable &t, uint64_t key, unsigned long long count,
                                                 int64_t *status) {
    uint64_t slot = table_home(key, t.mask);
    for (uint64_t probes = 0; probes <= t.mask; ++probes) {
        unsigned long long cur = ld_relaxed(reinterpret_cast<const uint64_t *>(t.keys + slot));
        uint32_t claimed = 0;
        if (cur == kTableEmpty) {
            cur = atomicCAS(t.keys + slot, kTableEmpty, (unsigned long long)key);
            if (cur == kTableEmpty) { cur = key; claimed = 1; }
        }
        if (cur == key) {
            atomicAdd(t.counts + slot, count);
            return claimed;
        }
        slot = (slot + 1) & t.mask;
    }
    atomicExch((unsigned long long *)&status[BNPK_ST_TABLE_FULL], 1ull);
    return 0;
}

struct HistTarget {
    unsigned long long *global;  // int64 table in HBM/L2
    uint32_t *smem;              // privatised table (or nullptr)
    uint64_t n_bins;
    uint64_t mask;               // n_bins-1 when n_bins is a power of two, else 0
    unsigned long long delta;    // +1, or -1 for the un-count of an incomplete record
    uint64_t canon_xor;          // != 0: count min(h, reverse-complement hash) (see canonical_hash)
};

template <bool SMEM>
__device__ __forceinline__ void hist_add(const HistTarget &t, uint64_t value) {
    const uint64_t b = t.mask ? (value & t.mask) : (value % t.n_bins);
    if constexpr (SMEM)
        atomicAdd(t.smem + (uint32_t)b, 1u);
    else
        atomicAdd(t.global + b, t.delta);
}

// first invalid byte in [from, to) (relative to unit 0), -1 if all valid; s_bad[u] = the invalid-byte mask encode_unit
// gave unit u.  Warp-wide.
__device__ __forceinline__ int find_invalid(const uint32_t *s_bad, int from, int to, int lane) {
    if (to <= from) return -1;
    int unit0 = from >> 4;
    const int last_unit = (to + 15) >> 4;
    for (; unit0 < last_unit; unit0 += 32) {
        const int u = unit0 + lane;
        uint32_t bad = 0;
        if (u < last_unit) {
            bad = s_bad[u];
            if (u == (from >> 4)) bad &= 0xFFFFu << (from & 15);
            if (u == ((to - 1) >> 4)) bad &= 0xFFFFu >> (15 - ((to - 1) & 15));
        }
        const unsigned b = __ballot_sync(0xffffffffu, bad != 0);
        if (b) {
            const int src = __ffs(b) - 1;
            const int pos = (u << 4) + __ffs(bad) - 1;
            return __shfl_sync(0xffffffffu, pos, src);
        }
    }
    return -1;
}

// k-mers / minimizers of one staged row -> histogram.  Warp-wide.  Returns values counted by
// this lane.  `b0` = tile-relative byte of the row's first base, L = row length.
template <bool SMEM_HIST, bool MINIMIZER>
__device__ __forceinline__ uint32_t row_count(const uint32_t *s_codes, int b0, int L, int k, int window,
                                              const HistTarget &ht, int lane) {
    uint32_t produced = 0;
    const uint64_t kmask = (k == 32) ? ~0ull : ((1ull << (2 * k)) - 1);
    if constexpr (!MINIMIZER) {
        const int npos = L - k + 1;
        // fast path: the bin index only needs the low 32 bits of the window
        if (ht.mask && ht.mask <= 0xFFFFFFFFull && !ht.canon_xor) {
            const uint32_t m32 = (uint32_t)(ht.mask & kmask);
            for (int i = lane; i < npos; i += 32) {
                const uint32_t lo = stream_lo32(s_codes, (uint32_t)(b0 + i)) & m32;
                if constexpr (SMEM_HIST) atomicAdd(ht.smem + lo, 1u);
                else atomicAdd(ht.global + lo, ht.delta);
                ++produced;
            }
        } else {
            for (int i = lane; i < npos; i += 32) {
                uint64_t h = stream_64(s_codes, (uint32_t)(b0 + i)) & kmask;
                if (ht.canon_xor) h = canonical_hash(h, k, ht.canon_xor);
                hist_add<SMEM_HIST>(ht, h);
                ++produced;
            }
        }
    } else {
        const int w = window - k + 1;           // k-mers per window (minimizers.py:52)
        const int nout = L - window + 1;        // windows in the row
        const int nh = L - k + 1;               // hashes in the row
        if (w <= 32) {
            const int step = 32 - (w - 1);
            for (int base = 0; base < nout; base += step) {
                const int p = base + lane;
                uint64_t h = ~0ull;
                if (p < nh) h = stream_64(s_codes, (uint32_t)(b0 + p)) & kmask;
                const uint64_t m = warp_sliding_min(h, w);
                if (lane < step && p < nout) { hist_add<SMEM_HIST>(ht, m); ++produced; }
            }
        } else {
            for (int j = lane; j < nout; j += 32) {
                uint64_t m = ~0ull;
                for (int i = 0; i < w; ++i) {
                    const uint64_t h = stream_64(s_codes, (uint32_t)(b0 + j + i)) & kmask;
                    m = h < m ? h : m;
                }
                hist_add<SMEM_HIST>(ht, m);
                ++produced;
            }
        }
    }
    return produced;
}

}  // namespace bnpk
