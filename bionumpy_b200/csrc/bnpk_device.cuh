// bnpk_device.cuh -- shared device helpers for the sm_90a k-mer hot path.
//
// Data model (see DESIGN.md):
//   every 16-byte unit of the raw chunk is turned, in registers, into
//     codes32 : 2 bits per byte  (byte j of the unit at bits 2j)  -> a contiguous 2-bit stream
//     flags32 : low 16 bits = "byte is '\n'", high 16 bits = "byte is a valid base"
//   and only those 8 bytes per unit are kept in shared memory.  A k-mer starting at byte b is
//   the 2k-bit field at bit 2b of the packed stream (first base in the lowest bits), which is
//   exactly the reference hash sum_j code[i+j]*4^j (sequence/kmers.py:105-126).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
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

__device__ __forceinline__ uint64_t warp_sum_u64(uint64_t v) {
#pragma unroll
    for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// Decoupled look-back (single-pass chained scan).  Called by one full warp.  Publishes this
// tile's aggregate, walks back over predecessors until an inclusive prefix is found, publishes
// the tile's inclusive prefix and returns the exclusive one.  Tiles are handed out in
// increasing order by an atomic ticket, so every predecessor is already running (or done).
// The walk keeps kLookbackDepth windows of 32 predecessors in flight per round trip.
constexpr int kLookbackDepth = 4;
__device__ __forceinline__ uint64_t lookback_exclusive(uint64_t *state, int64_t tile, uint64_t aggregate, int lane) {
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
                excl += warp_sum_u64(v);
            }
        }
        if (done) break;
        idx -= 32 * kLookbackDepth;
    }
    if (lane == 0) st_relaxed(state + tile, kFlagPrefix | ((excl + aggregate) & kValueMask));
    return excl;
}

// ---------------------------------------------------------------------------------------------
// byte -> code / flag transforms, four bytes at a time
// ---------------------------------------------------------------------------------------------
// gather bit 0 of each byte into a nibble (bits 0..3)
__device__ __forceinline__ uint32_t bytes_lsb_to_nibble(uint32_t m01) {
    return ((m01 & 0x01010101u) * 0x00204081u >> 21) & 0xFu;
}
// gather the low 2 bits of each byte into 8 bits
__device__ __forceinline__ uint32_t bytes_2bit_to_byte(uint32_t x03) {
    return (x03 * 0x01041040u) >> 24;
}

template <int ENC>
__device__ __forceinline__ void encode_word(uint32_t w, const uint8_t *s_lut, uint32_t &code8, uint32_t &valid4) {
    if constexpr (ENC == BNPK_ENC_ASCII_ACGT || ENC == BNPK_ENC_ASCII_ACTG) {
        uint32_t x;
        if constexpr (ENC == BNPK_ENC_ASCII_ACGT)
            x = ((w >> 1) ^ (w >> 2)) & 0x03030303u;  // A0 C1 G2 T3
        else
            x = (w >> 1) & 0x03030303u;                // A0 C1 T2 G3
        code8 = bytes_2bit_to_byte(x);
        const uint32_t u = w | 0x20202020u;            // fold case (alphabet_encoding.py:24-28)
        const uint32_t eq = __vcmpeq4(u, 0x61616161u) | __vcmpeq4(u, 0x63636363u) |
                            __vcmpeq4(u, 0x67676767u) | __vcmpeq4(u, 0x74747474u);
        valid4 = bytes_lsb_to_nibble(eq);
    } else if constexpr (ENC == BNPK_ENC_CODES) {
        code8 = bytes_2bit_to_byte(w & 0x03030303u);
        valid4 = bytes_lsb_to_nibble(__vcmpeq4(w & 0xFCFCFCFCu, 0u));
    } else {
        uint32_t c = 0, v = 0;
#pragma unroll
        for (int b = 0; b < 4; ++b) {
            const uint32_t code = s_lut[(w >> (8 * b)) & 0xFFu];
            c |= (code & 3u) << (2 * b);
            v |= (code < 4u ? 1u : 0u) << b;
        }
        code8 = c;
        valid4 = v;
    }
}

// one 16-byte unit -> (codes32, flags32)
template <int ENC>
__device__ __forceinline__ void encode_unit(const uint4 q, const uint8_t *s_lut, uint32_t &codes, uint32_t &flags) {
    uint32_t c0, c1, c2, c3, v0, v1, v2, v3;
    encode_word<ENC>(q.x, s_lut, c0, v0);
    encode_word<ENC>(q.y, s_lut, c1, v1);
    encode_word<ENC>(q.z, s_lut, c2, v2);
    encode_word<ENC>(q.w, s_lut, c3, v3);
    codes = c0 | (c1 << 8) | (c2 << 16) | (c3 << 24);
    const uint32_t nl = bytes_lsb_to_nibble(__vcmpeq4(q.x, 0x0A0A0A0Au)) |
                        (bytes_lsb_to_nibble(__vcmpeq4(q.y, 0x0A0A0A0Au)) << 4) |
                        (bytes_lsb_to_nibble(__vcmpeq4(q.z, 0x0A0A0A0Au)) << 8) |
                        (bytes_lsb_to_nibble(__vcmpeq4(q.w, 0x0A0A0A0Au)) << 12);
    flags = nl | ((v0 | (v1 << 4) | (v2 << 8) | (v3 << 12)) << 16);
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
            const uint4 q = load_unit_guarded(base, n, ub);
            m = bytes_lsb_to_nibble(__vcmpeq4(q.x, 0x0A0A0A0Au)) | (bytes_lsb_to_nibble(__vcmpeq4(q.y, 0x0A0A0A0Au)) << 4) |
                (bytes_lsb_to_nibble(__vcmpeq4(q.z, 0x0A0A0A0Au)) << 8) | (bytes_lsb_to_nibble(__vcmpeq4(q.w, 0x0A0A0A0Au)) << 12);
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

// first invalid byte in [from, to) (tile-relative), -1 if all valid.  Warp-wide.
__device__ __forceinline__ int find_invalid(const uint32_t *s_flags, int from, int to, int lane) {
    if (to <= from) return -1;
    int unit0 = from >> 4;
    const int last_unit = (to + 15) >> 4;
    for (; unit0 < last_unit; unit0 += 32) {
        const int u = unit0 + lane;
        uint32_t bad = 0;
        if (u < last_unit) {
            bad = (~(s_flags[u] >> 16)) & 0xFFFFu;
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
