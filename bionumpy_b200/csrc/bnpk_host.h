// bnpk_host.h -- host-side glue shared by the translation units of libbnpk.so
#pragma once
#include <algorithm>
#include <atomic>
#include <cstdio>
#include <cstring>
#include <type_traits>
#include "bnpk_device.cuh"

namespace bnpk {

extern std::atomic<uint64_t> g_launches;
int set_err(int code, const char *msg);
int cuda_fail(cudaError_t e, const char *what);
int sm_count();
// cudaFuncAttributeMaxDynamicSharedMemorySize is a per-device attribute: set it once per (kernel, device)
int ensure_dyn_smem(const void *kernel, int bytes);
#define BNPK_DYN_SMEM(kern, bytes)                                            \
    do {                                                                      \
        int rc__ = ::bnpk::ensure_dyn_smem((const void *)(kern), (int)(bytes)); \
        if (rc__) return rc__;                                                \
    } while (0)

#define BNPK_CUDA(expr)                                             \
    do {                                                            \
        cudaError_t e__ = (expr);                                   \
        if (e__ != cudaSuccess) return ::bnpk::cuda_fail(e__, #expr); \
    } while (0)

// optional per-launch timing of the dominant (tile) kernel, see bnpk_profile_* in bnpk.h
void profile_before(cudaStream_t st);
void profile_after(cudaStream_t st);

// Calls f(std::integral_constant<int, ENC>{}) with the BNPK_ENC_* that enc_mode names; any other value is refused.
template <typename F>
int with_enc(int enc_mode, F &&f) {
    switch (enc_mode) {
        case BNPK_ENC_ASCII_ACGT: return f(std::integral_constant<int, BNPK_ENC_ASCII_ACGT>{});
        case BNPK_ENC_ASCII_ACTG: return f(std::integral_constant<int, BNPK_ENC_ASCII_ACTG>{});
        case BNPK_ENC_CODES: return f(std::integral_constant<int, BNPK_ENC_CODES>{});
        case BNPK_ENC_LUT: return f(std::integral_constant<int, BNPK_ENC_LUT>{});
    }
    return set_err(BNPK_E_BADARG, "bad enc_mode");
}

// Whether enc_mode can give the codes of an alphabet of alphabet_size letters: the ASCII encodings only give four-letter
// codes, raw bytes (alphabet_size 256) are their own codes, and BNPK_ENC_LUT reads lut256.
inline int check_enc(int enc_mode, const uint8_t *lut256, int alphabet_size) {
    if (enc_mode < 0 || enc_mode > 3) return set_err(BNPK_E_BADARG, "bad enc_mode");
    if (alphabet_size != 4 && enc_mode != BNPK_ENC_LUT && enc_mode != BNPK_ENC_CODES)
        return set_err(BNPK_E_BADARG, "alphabets that are not four letters take BNPK_ENC_LUT or BNPK_ENC_CODES");
    if (alphabet_size == 256 && enc_mode != BNPK_ENC_CODES)
        return set_err(BNPK_E_BADARG, "raw bytes (alphabet_size 256) take BNPK_ENC_CODES");
    if (enc_mode == BNPK_ENC_LUT && !lut256) return set_err(BNPK_E_BADARG, "lut256 required");
    return 0;
}

// The grid of a grid-stride kernel: the CTAs its work asks for, at most ctas_per_sm on every SM, and at least one.
inline unsigned grid_cap(size_t ctas_wanted, int ctas_per_sm) {
    return (unsigned)std::max<size_t>(1, std::min(ctas_wanted, (size_t)sm_count() * ctas_per_sm));
}

// kern<<<grid, block, smem, st>>>(args...), counted in bnpk_launch_count; `profiled` times it for bnpk_profile_read.
template <typename... P, typename... A>
int launch(const char *name, void (*kern)(P...), unsigned grid, int block, size_t smem, cudaStream_t st, bool profiled,
           const A &...args) {
    if (profiled) profile_before(st);
    kern<<<grid, block, smem, st>>>(args...);
    if (profiled) profile_after(st);
    g_launches.fetch_add(1, std::memory_order_relaxed);
    const cudaError_t e = cudaGetLastError();
    return e == cudaSuccess ? 0 : cuda_fail(e, name);
}

// A kernel that takes every CTA slot its shared memory leaves: raises its dynamic shared-memory limit to smem_max,
// refuses with BNPK_E_BINS and `misfit` when not one CTA of `smem` bytes fits an SM, and launches as many CTAs as are
// resident at once, at most ctas_wanted (none for no work).
template <typename... P, typename... A>
int launch_resident(const char *name, const char *misfit, void (*kern)(P...), size_t ctas_wanted, int block,
                    size_t smem, size_t smem_max, cudaStream_t st, bool profiled, const A &...args) {
    BNPK_DYN_SMEM(kern, smem_max);
    int per_sm = 1;
    BNPK_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, block, smem));
    if (per_sm < 1) return set_err(BNPK_E_BINS, misfit);
    if (ctas_wanted == 0) return 0;
    return launch(name, kern, grid_cap(ctas_wanted, per_sm), block, smem, st, profiled, args...);
}

// The workspace of a single-pass scan of n items (bnpk_device.cuh) that runs n_scans look-backs: sets n_tiles (at
// least one), refuses a workspace smaller than the header and n_scans states per tile, and zeroes that much on st.
inline int scan_workspace(size_t n, int n_scans, void *workspace, size_t workspace_bytes, cudaStream_t st,
                          size_t &n_tiles) {
    n_tiles = std::max<size_t>((n + kScanTile - 1) / kScanTile, 1);
    const size_t need = (kWsHeaderWords + n_scans * n_tiles) * sizeof(uint64_t);
    if (workspace_bytes < need) return set_err(BNPK_E_WORKSPACE, "workspace too small");
    BNPK_CUDA(cudaMemsetAsync(workspace, 0, need, st));
    return 0;
}

size_t tile_workspace_bytes(size_t n);
bool use_smem_hist(int64_t n_bins, int hist_mode);

int chunk_kmer_count_impl(const uint8_t *chunk, size_t n, size_t slice_begin, size_t slice_end, int final_slice,
                          int lpe, uint8_t header_char, int check_plus, int trim_cr, int enc_mode,
                          const uint8_t *lut256, int k, int window, int64_t n_bins, int hist_mode, int64_t *hist,
                          int64_t *status, void *workspace, size_t workspace_bytes, cudaStream_t st);

int line_split_impl(const uint8_t *chunk, size_t n, int lpe, int field_line, int start_offset, uint8_t header_char,
                    int check_plus, int trim_cr, int64_t *starts, int32_t *lens, size_t max_rows, int64_t *status,
                    void *workspace, size_t workspace_bytes, cudaStream_t st);

// after the last slice of a fused count: long (deferred) rows + un-count of the sequence line
// of a trailing incomplete entry
int count_fixups_impl(const uint8_t *chunk, size_t n, int lpe, int enc_mode, const uint8_t *lut256, int k,
                      int window, int64_t n_bins, int64_t *hist, int64_t *status, const uint64_t *deferred_count,
                      const uint64_t *deferred, size_t deferred_cap, cudaStream_t st);

}  // namespace bnpk
