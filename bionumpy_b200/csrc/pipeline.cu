// pipeline.cu -- host-buffer entry point: slice-wise H2D copy overlapped with the fused count.
// This is what replaces CupyFileReader._get_buffer's cp.asanyarray(chunk)
// (bionumpy/cupy_compatible/parser.py:11-17) followed by the K6 chain.
#include <vector>
#include "bnpk_host.h"

struct bnpk_pipeline {
    int device = 0;
    size_t capacity = 0, slice_bytes = 0;
    uint8_t *d_chunk = nullptr;
    void *d_ws = nullptr;
    size_t ws_bytes = 0;
    int64_t *d_status = nullptr;
    uint8_t *d_lut = nullptr;
    int64_t *h_status = nullptr;  // pinned
    cudaStream_t copy_stream = nullptr, compute_stream = nullptr;
    std::vector<cudaEvent_t> events;
    cudaEvent_t ev_in = nullptr;       // the caller's stream at the time of the call
};

using namespace bnpk;

extern "C" {

int bnpk_pipeline_create(bnpk_pipeline **out, size_t capacity_bytes, size_t slice_bytes) {
    if (!out || capacity_bytes == 0) return set_err(BNPK_E_BADARG, "bad pipeline arguments");
    if (slice_bytes == 0) slice_bytes = (size_t)64 << 20;
    slice_bytes = (slice_bytes + kTileBytes - 1) / kTileBytes * kTileBytes;
    bnpk_pipeline *p = new bnpk_pipeline();
    *out = p;
    BNPK_CUDA(cudaGetDevice(&p->device));
    p->capacity = capacity_bytes;
    p->slice_bytes = slice_bytes;
    p->ws_bytes = tile_workspace_bytes(capacity_bytes);
    BNPK_CUDA(cudaMalloc(&p->d_chunk, capacity_bytes + 64));
    BNPK_CUDA(cudaMalloc(&p->d_ws, p->ws_bytes));
    BNPK_CUDA(cudaMalloc(&p->d_status, BNPK_ST_WORDS * sizeof(int64_t)));
    BNPK_CUDA(cudaMalloc(&p->d_lut, 256));
    BNPK_CUDA(cudaMallocHost(&p->h_status, BNPK_ST_WORDS * sizeof(int64_t)));
    BNPK_CUDA(cudaStreamCreateWithFlags(&p->copy_stream, cudaStreamNonBlocking));
    BNPK_CUDA(cudaStreamCreateWithFlags(&p->compute_stream, cudaStreamNonBlocking));
    const size_t n_slices = (capacity_bytes + slice_bytes - 1) / slice_bytes;
    p->events.resize(n_slices);
    for (auto &e : p->events) BNPK_CUDA(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
    BNPK_CUDA(cudaEventCreateWithFlags(&p->ev_in, cudaEventDisableTiming));
    return 0;
}

void bnpk_pipeline_destroy(bnpk_pipeline *p) {
    if (!p) return;
    for (auto &e : p->events) cudaEventDestroy(e);
    if (p->ev_in) cudaEventDestroy(p->ev_in);
    if (p->copy_stream) cudaStreamDestroy(p->copy_stream);
    if (p->compute_stream) cudaStreamDestroy(p->compute_stream);
    cudaFree(p->d_chunk);
    cudaFree(p->d_ws);
    cudaFree(p->d_status);
    cudaFree(p->d_lut);
    cudaFreeHost(p->h_status);
    delete p;
}

int bnpk_pipeline_kmer_count_host_on(bnpk_pipeline *p, const uint8_t *chunk_host, size_t n, int lines_per_entry,
                                     uint8_t header_char, int check_plus, int trim_cr, int enc_mode,
                                     const uint8_t *lut256_host, int k, int window_size, int64_t n_bins, int hist_mode,
                                     int64_t *hist, int64_t *status_host, void *stream) {
    if (!p || (!chunk_host && n) || !status_host) return set_err(BNPK_E_BADARG, "null argument");
    if (n > p->capacity) return set_err(BNPK_E_BADARG, "chunk larger than the pipeline capacity");
    cudaStream_t cs = p->compute_stream;
    // the private streams do not synchronise with anybody: order the count after what the caller has queued
    // (the kernel or memset that produced `hist`)
    BNPK_CUDA(cudaEventRecord(p->ev_in, (cudaStream_t)stream));
    BNPK_CUDA(cudaStreamWaitEvent(cs, p->ev_in, 0));
    if (int rc = bnpk_status_init(p->d_status, cs)) return rc;
    if (enc_mode == BNPK_ENC_LUT) {
        if (!lut256_host) return set_err(BNPK_E_BADARG, "lut256 required");
        BNPK_CUDA(cudaMemcpyAsync(p->d_lut, lut256_host, 256, cudaMemcpyHostToDevice, cs));
    }
    const size_t n_slices = n ? (n + p->slice_bytes - 1) / p->slice_bytes : 0;
    for (size_t s = 0; s < n_slices; ++s) {
        const size_t b = s * p->slice_bytes, e = std::min(n, b + p->slice_bytes);
        BNPK_CUDA(cudaMemcpyAsync(p->d_chunk + b, chunk_host + b, e - b, cudaMemcpyHostToDevice, p->copy_stream));
        BNPK_CUDA(cudaEventRecord(p->events[s], p->copy_stream));
        BNPK_CUDA(cudaStreamWaitEvent(cs, p->events[s], 0));
        const int rc = chunk_kmer_count_impl(p->d_chunk, n, b, e, s + 1 == n_slices, lines_per_entry, header_char,
                                             check_plus, trim_cr, enc_mode, p->d_lut, k, window_size, n_bins,
                                             hist_mode, hist, p->d_status, p->d_ws, p->ws_bytes, cs);
        if (rc) return rc;
    }
    BNPK_CUDA(cudaMemcpyAsync(p->h_status, p->d_status, BNPK_ST_WORDS * sizeof(int64_t), cudaMemcpyDeviceToHost, cs));
    BNPK_CUDA(cudaStreamSynchronize(cs));
    memcpy(status_host, p->h_status, BNPK_ST_WORDS * sizeof(int64_t));
    return 0;
}

int bnpk_pipeline_kmer_count_host(bnpk_pipeline *p, const uint8_t *chunk_host, size_t n, int lines_per_entry,
                                  uint8_t header_char, int check_plus, int trim_cr, int enc_mode,
                                  const uint8_t *lut256_host, int k, int window_size, int64_t n_bins, int hist_mode,
                                  int64_t *hist, int64_t *status_host) {
    return bnpk_pipeline_kmer_count_host_on(p, chunk_host, n, lines_per_entry, header_char, check_plus, trim_cr, enc_mode,
                                            lut256_host, k, window_size, n_bins, hist_mode, hist, status_host, nullptr);
}

}  // extern "C"
