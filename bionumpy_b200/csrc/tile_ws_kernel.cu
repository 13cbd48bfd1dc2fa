// tile_ws_kernel.cu -- the two builds of the warp-specialised fused count (tile_ws_kernel.inl)
#include "tile_common.cuh"

// k-mer counts: the dominant kernel of the hot path
#define BNPK_WS_NAMESPACE ws
#define BNPK_WS_NS 8
#define BNPK_WS_SG 2
#define BNPK_WS_RW 8
#define BNPK_WS_MINZ 0
#define BNPK_WS_LAUNCH launch_ws_count
#include "tile_ws_kernel.inl"
#undef BNPK_WS_NAMESPACE
#undef BNPK_WS_NS
#undef BNPK_WS_SG
#undef BNPK_WS_RW
#undef BNPK_WS_MINZ
#undef BNPK_WS_LAUNCH

// minimizer counts (windows of up to 12 k-mers, CTA-private table)
#define BNPK_WS_NAMESPACE wsm
#define BNPK_WS_NS 4       // the slots are held for the front end and the encoding only (rows are staged), see kStageU
#define BNPK_WS_SG 1       // the row warps bound this build: one scan group is enough, and sixteen row warps (80 registers
#define BNPK_WS_RW 16      // per thread, no spills; on H100 16 row warps beat 14 and 12 by 8 and 13 %)
#define BNPK_WS_MINZ 1
#define BNPK_WS_LAUNCH launch_wsm_count
#include "tile_ws_kernel.inl"

namespace bnpk {
// Both builds count into a CTA-private table of at most kMaxBins bins and stage the chunk by bulk copies, which need a
// 16-byte-aligned chunk; tile indices stay in 31 bits.
static bool ws_common_eligible(const TileArgs &a, bool smem_hist) {
    if (!smem_hist || a.n_bins > (uint64_t)ws::kMaxBins) return false;
    if ((reinterpret_cast<uintptr_t>(a.chunk) & 15) != 0) return false;
    return a.tile_end <= 0x7FFFFFF0ll && a.n >= 16;
}
// k-mer counts
bool ws_count_eligible(const TileArgs &a, bool smem_hist) { return a.window == 0 && ws_common_eligible(a, smem_hist); }
// minimizer counts with windows of at most kMinzW k-mers
bool wsm_count_eligible(const TileArgs &a, bool smem_hist) {
    return a.window != 0 && a.window - a.k + 1 <= wsm::kMinzW && ws_common_eligible(a, smem_hist);
}
}  // namespace bnpk
