// torch_ops.cpp -- TORCH_LIBRARY(bnpk, ...): the k-mer hot path as PyTorch dispatcher ops.
//
// north_star: "the ragged-array and k-mer kernels bound through PyTorch's C++/CUDA extension ABI".  This file is that
// binding: a thin layer over the C-ABI of libbnpk.so (include/bnpk.h), built into libbnpk_torch.so.  Every op
//   * runs on the device of its tensors (CUDAGuard) and on torch's current stream of that device,
//   * allocates its outputs, its status block and its look-back workspace from torch's caching allocator PER CALL --
//     so two streams (or two threads) never share scratch state, and a buffer is reused only in stream order,
//   * never synchronises: the status block comes back as a tensor, the Python layer reads it when it wants to.
// It replaces the reference's `bnp.set_backend(cupy)` seam (bionumpy/__init__.py:47-94) for this path; the functions
// each op stands for are named in include/bnpk.h.
#include <ATen/cuda/CUDAContext.h>
#include <c10/cuda/CUDAGuard.h>
#include <torch/library.h>
#include <torch/torch.h>

#include "../../include/bnpk.h"

namespace {

using torch::Tensor;

void check(int rc, const char *what) {
    TORCH_CHECK(rc == 0, "bnpk::", what, ": ", bnpk_last_error(), " (code ", rc, ")");
}
const uint8_t *u8(const Tensor &t) { return t.defined() && t.numel() ? t.data_ptr<uint8_t>() : nullptr; }
// t is a contiguous CUDA tensor of dtype st, on the device of `on` when that is given: a kernel reads every pointer it
// gets on the device it runs on.
void need(const Tensor &t, c10::ScalarType st, const char *name, const Tensor &on = Tensor()) {
    TORCH_CHECK(t.is_cuda() && t.is_contiguous() && t.scalar_type() == st, "bnpk: ", name,
                " must be a contiguous CUDA tensor of the right dtype");
    TORCH_CHECK(!on.defined() || t.device() == on.device(), "bnpk: ", name, " is on ", t.device(), ", not on ",
                on.device());
}
// an optional 256-byte table: the kernels read all of it
const uint8_t *need_lut(const c10::optional<Tensor> &lut, const char *name, const Tensor &on) {
    if (!lut) return nullptr;
    need(*lut, torch::kUInt8, name, on);
    TORCH_CHECK(lut->numel() == 256, "bnpk: ", name, " must have 256 entries");
    return lut->data_ptr<uint8_t>();
}
// out_offsets[r] for the rows r < n_rows, and the total at n_rows
const int64_t *need_offsets(const Tensor &offsets, size_t n_rows, const Tensor &on) {
    need(offsets, torch::kInt64, "offsets", on);
    TORCH_CHECK((size_t)offsets.numel() >= n_rows + 1, "bnpk: offsets need one entry per row and the total");
    return offsets.data_ptr<int64_t>();
}
void *cur_stream(const Tensor &t) { return (void *)at::cuda::getCurrentCUDAStream(t.get_device()).stream(); }
Tensor new_status(const Tensor &like) {
    Tensor st = torch::empty({BNPK_ST_WORDS}, like.options().dtype(torch::kInt64));
    check(bnpk_status_init(st.data_ptr<int64_t>(), cur_stream(like)), "status_init");
    return st;
}
Tensor new_workspace(const Tensor &like, size_t n) {
    return torch::empty({(int64_t)bnpk_tile_workspace_bytes(n)}, like.options().dtype(torch::kUInt8));
}

// The rows of a row op: bytes base[starts[r], starts[r] + lens[r]) for r < n_rows, and the op's 256-byte lut (or
// null).  call(fn, more...) is fn(base, base_bytes, starts, lens, n_rows, more...), the head of every bnpk_rows_*.
struct Rows {
    const uint8_t *base;
    size_t base_bytes;
    const int64_t *starts;
    const int32_t *lens;
    size_t n_rows;
    const uint8_t *lut;
    template <typename F, typename... A>
    int call(F fn, A... more) const { return fn(base, base_bytes, starts, lens, n_rows, more...); }
};

// base uint8, starts int64 and lens int32 of one length, and lut uint8[256] or None: contiguous CUDA tensors, all on
// the device of `on` (default: base's).
Rows need_rows(const Tensor &base, const Tensor &starts, const Tensor &lens, const c10::optional<Tensor> &lut,
               const Tensor &on = Tensor()) {
    const Tensor &dev = on.defined() ? on : base;
    need(base, torch::kUInt8, "base", dev);
    need(starts, torch::kInt64, "starts", dev);
    need(lens, torch::kInt32, "lens", dev);
    TORCH_CHECK(starts.numel() == lens.numel(), "bnpk: starts and lens differ in length");
    return Rows{u8(base), (size_t)base.numel(), starts.data_ptr<int64_t>(), lens.data_ptr<int32_t>(),
                (size_t)lens.numel(), need_lut(lut, "lut", dev)};
}

// K6: chunk bytes -> histogram (accumulated into hist).  Returns the status block.
Tensor chunk_kmer_count(const Tensor &chunk, int64_t k, int64_t window_size, Tensor hist, int64_t lines_per_entry,
                        int64_t header_char, bool check_plus, int64_t trim_cr, int64_t enc_mode,
                        const c10::optional<Tensor> &lut, int64_t hist_mode) {
    need(chunk, torch::kUInt8, "chunk");
    need(hist, torch::kInt64, "hist", chunk);
    const uint8_t *l = need_lut(lut, "lut", chunk);
    c10::cuda::CUDAGuard guard(chunk.device());
    Tensor status = new_status(chunk);
    const size_t n = (size_t)chunk.numel();
    Tensor ws = new_workspace(chunk, n);
    check(bnpk_chunk_kmer_count(chunk.data_ptr<uint8_t>(), n, 0, n, 1, (int)lines_per_entry, (uint8_t)header_char,
                                check_plus, (int)trim_cr, (int)enc_mode, l, (int)k, (int)window_size, hist.numel(),
                                (int)hist_mode, hist.data_ptr<int64_t>(), status.data_ptr<int64_t>(), ws.data_ptr<uint8_t>(),
                                (size_t)ws.numel(), cur_stream(chunk)),
          "chunk_kmer_count");
    return status;
}

// K1: (starts int64[max_rows], lens int32[max_rows], status)
std::tuple<Tensor, Tensor, Tensor> line_split(const Tensor &chunk, int64_t lines_per_entry, int64_t field_line,
                                              int64_t start_offset, int64_t header_char, bool check_plus,
                                              int64_t trim_cr, int64_t max_rows) {
    need(chunk, torch::kUInt8, "chunk");
    c10::cuda::CUDAGuard guard(chunk.device());
    Tensor starts = torch::empty({max_rows}, chunk.options().dtype(torch::kInt64));
    Tensor lens = torch::empty({max_rows}, chunk.options().dtype(torch::kInt32));
    Tensor status = new_status(chunk);
    const size_t n = (size_t)chunk.numel();
    Tensor ws = new_workspace(chunk, n);
    check(bnpk_line_split(chunk.data_ptr<uint8_t>(), n, (int)lines_per_entry, (int)field_line, (int)start_offset,
                          (uint8_t)header_char, check_plus, (int)trim_cr, starts.data_ptr<int64_t>(),
                          lens.data_ptr<int32_t>(), (size_t)max_rows, status.data_ptr<int64_t>(), ws.data_ptr<uint8_t>(),
                          (size_t)ws.numel(), cur_stream(chunk)),
          "line_split");
    return {starts, lens, status};
}

Tensor row_offsets(const Tensor &lens, int64_t shrink) {
    need(lens, torch::kInt32, "lens");
    c10::cuda::CUDAGuard guard(lens.device());
    Tensor out = torch::empty({lens.numel() + 1}, lens.options().dtype(torch::kInt64));
    Tensor ws = new_workspace(lens, (size_t)std::max<int64_t>(lens.numel(), 1));
    check(bnpk_row_offsets(lens.data_ptr<int32_t>(), (size_t)lens.numel(), (int)shrink, out.data_ptr<int64_t>(),
                           ws.data_ptr<uint8_t>(), (size_t)ws.numel(), cur_stream(lens)),
          "row_offsets");
    return out;
}

// K2: codes uint8[total] (total = offsets[-1], given by the caller: no sync here)
std::tuple<Tensor, Tensor> rows_encode(const Tensor &base, const Tensor &starts, const Tensor &lens, int64_t enc_mode,
                                       const c10::optional<Tensor> &lut, const Tensor &offsets, int64_t total) {
    const Rows r = need_rows(base, starts, lens, lut);
    const int64_t *offs = need_offsets(offsets, r.n_rows, base);
    c10::cuda::CUDAGuard guard(base.device());
    Tensor out = torch::empty({total}, base.options());
    Tensor status = new_status(base);
    check(r.call(bnpk_rows_encode, (int)enc_mode, r.lut, offs, out.data_ptr<uint8_t>(), status.data_ptr<int64_t>(),
                 cur_stream(base)),
          "rows_encode");
    return {out, status};
}

// K3 / K4: hashes or minimizers int64[total]
std::tuple<Tensor, Tensor> rows_kmer_hash(const Tensor &base, const Tensor &starts, const Tensor &lens, int64_t enc_mode,
                                          const c10::optional<Tensor> &lut, int64_t k, int64_t window_size,
                                          int64_t complement_xor, const Tensor &offsets, int64_t total) {
    const Rows r = need_rows(base, starts, lens, lut);
    const int64_t *offs = need_offsets(offsets, r.n_rows, base);
    TORCH_CHECK(window_size == 0 || complement_xor == 0, "bnpk: minimizers are not canonical (complement_xor must be 0)");
    c10::cuda::CUDAGuard guard(base.device());
    Tensor out = torch::empty({total}, base.options().dtype(torch::kInt64));
    Tensor status = new_status(base);
    int64_t *o = out.data_ptr<int64_t>(), *st = status.data_ptr<int64_t>();
    int rc;
    if (window_size)
        rc = r.call(bnpk_rows_minimizers, (int)enc_mode, r.lut, (int)k, (int)window_size, offs, o, st, cur_stream(base));
    else if (complement_xor)
        rc = r.call(bnpk_rows_kmer_hash_canonical, (int)enc_mode, r.lut, (int)k, (int)complement_xor, offs, o, st,
                    cur_stream(base));
    else
        rc = r.call(bnpk_rows_kmer_hash, (int)enc_mode, r.lut, (int)k, offs, o, st, cur_stream(base));
    check(rc, "rows_kmer_hash");
    return {out, status};
}

// K3/K4 + K5 on a ragged view (accumulates into hist)
Tensor rows_kmer_count(const Tensor &base, const Tensor &starts, const Tensor &lens, int64_t enc_mode,
                       const c10::optional<Tensor> &lut, int64_t k, int64_t window_size, int64_t complement_xor,
                       Tensor hist, int64_t hist_mode) {
    const Rows r = need_rows(base, starts, lens, lut);
    need(hist, torch::kInt64, "hist", base);
    TORCH_CHECK(window_size == 0 || complement_xor == 0, "bnpk: minimizers are not canonical (complement_xor must be 0)");
    c10::cuda::CUDAGuard guard(base.device());
    Tensor status = new_status(base);
    int rc;
    if (complement_xor)
        rc = r.call(bnpk_rows_kmer_count_canonical, (int)enc_mode, r.lut, (int)k, (int)complement_xor, hist.numel(),
                    (int)hist_mode, hist.data_ptr<int64_t>(), status.data_ptr<int64_t>(), cur_stream(base));
    else
        rc = r.call(bnpk_rows_kmer_count, (int)enc_mode, r.lut, (int)k, (int)window_size, hist.numel(), (int)hist_mode,
                    hist.data_ptr<int64_t>(), status.data_ptr<int64_t>(), cur_stream(base));
    check(rc, "rows_kmer_count");
    return status;
}

// exact k-mer table: insert every k-mer of the rows (mutates keys, counts, n_used).  Returns the status block.
Tensor rows_kmer_table_insert(const Tensor &base, const Tensor &starts, const Tensor &lens, int64_t enc_mode,
                              const c10::optional<Tensor> &lut, int64_t k, int64_t complement_xor, Tensor keys,
                              Tensor counts, Tensor n_used) {
    const Rows r = need_rows(base, starts, lens, lut);
    need(keys, torch::kInt64, "keys", base);
    need(counts, torch::kInt64, "counts", base);
    need(n_used, torch::kInt64, "n_used", base);
    TORCH_CHECK(keys.numel() == counts.numel() && n_used.numel() == 1, "bnpk: keys/counts differ in length or n_used is not one word");
    c10::cuda::CUDAGuard guard(base.device());
    Tensor status = new_status(base);
    check(r.call(bnpk_rows_kmer_table_insert, (int)enc_mode, r.lut, (int)k, (int)complement_xor, keys.data_ptr<int64_t>(),
                 counts.data_ptr<int64_t>(), (size_t)keys.numel(), n_used.data_ptr<int64_t>(), status.data_ptr<int64_t>(),
                 cur_stream(base)),
          "rows_kmer_table_insert");
    return status;
}

Tensor rows_reverse_complement(const Tensor &base, const Tensor &starts, const Tensor &lens, const Tensor &lut,
                               const Tensor &offsets, int64_t total) {
    const Rows r = need_rows(base, starts, lens, lut);
    const int64_t *offs = need_offsets(offsets, r.n_rows, base);
    c10::cuda::CUDAGuard guard(base.device());
    Tensor out = torch::empty({total}, base.options());
    check(r.call(bnpk_rows_reverse_complement, r.lut, offs, out.data_ptr<uint8_t>(), cur_stream(base)),
          "rows_reverse_complement");
    return out;
}

// K7: motif scores float64[total] of matrix [motif_len, alphabet_size] (float64, on the device)
std::tuple<Tensor, Tensor> rows_pwm_scores(const Tensor &base, const Tensor &starts, const Tensor &lens, int64_t enc_mode,
                                           const c10::optional<Tensor> &lut, const Tensor &matrix, bool tail,
                                           const Tensor &offsets, int64_t total) {
    const Rows r = need_rows(base, starts, lens, lut);
    const int64_t *offs = need_offsets(offsets, r.n_rows, base);
    need(matrix, torch::kFloat64, "matrix", base);
    TORCH_CHECK(matrix.dim() == 2, "bnpk: matrix must be [motif_len, alphabet_size]");
    c10::cuda::CUDAGuard guard(base.device());
    Tensor out = torch::empty({total}, base.options().dtype(torch::kFloat64));
    Tensor status = new_status(base);
    check(r.call(bnpk_rows_pwm_scores, (int)enc_mode, r.lut, (int)matrix.size(1), matrix.data_ptr<double>(),
                 (int)matrix.size(0), (int)tail, offs, out.data_ptr<double>(), status.data_ptr<int64_t>(), cur_stream(base)),
          "rows_pwm_scores");
    return {out, status};
}

// K8: matches uint8[total] (1 = some sub-pattern matches there) of the column sets `sets` (int32 words, on the device)
std::tuple<Tensor, Tensor> rows_match(const Tensor &base, const Tensor &starts, const Tensor &lens, int64_t enc_mode,
                                      const c10::optional<Tensor> &lut, int64_t alphabet_size, const Tensor &sets,
                                      c10::IntArrayRef sub_lens, bool same, const Tensor &offsets, int64_t total) {
    const Rows r = need_rows(base, starts, lens, lut);
    const int64_t *offs = need_offsets(offsets, r.n_rows, base);
    need(sets, torch::kInt32, "sets", base);
    std::vector<int32_t> sl(sub_lens.begin(), sub_lens.end());
    c10::cuda::CUDAGuard guard(base.device());
    Tensor out = torch::empty({total}, base.options().dtype(torch::kUInt8));
    Tensor status = new_status(base);
    check(r.call(bnpk_rows_match, (int)enc_mode, r.lut, (int)alphabet_size,
                 reinterpret_cast<const uint32_t *>(sets.data_ptr<int32_t>()), sl.data(), (int)sl.size(),
                 (int)same, offs, out.data_ptr<uint8_t>(), status.data_ptr<int64_t>(), cur_stream(base)),
          "rows_match");
    return {out, status};
}

// K5 (accumulates into hist)
Tensor bincount(const Tensor &values, Tensor hist, int64_t hist_mode) {
    need(values, torch::kInt64, "values");
    need(hist, torch::kInt64, "hist", values);
    c10::cuda::CUDAGuard guard(values.device());
    Tensor status = new_status(values);
    check(bnpk_bincount(values.data_ptr<int64_t>(), (size_t)values.numel(), hist.numel(), (int)hist_mode,
                        hist.data_ptr<int64_t>(), status.data_ptr<int64_t>(), cur_stream(values)),
          "bincount");
    return status;
}

// Writers: fields = [name base, starts, lens, sequence base, starts, lens(, quality base, starts, lens)], luts = one
// optional 256-byte table per field, all on the device of the name base.  format_offsets returns (offsets int64[E+1],
// status); format_records writes bytes [out_begin, out_end) of the text (the caller reads offsets[-1] for the total: no
// sync here).
std::vector<bnpk_field> make_fields(const std::vector<Tensor> &fields, const std::vector<c10::optional<Tensor>> &luts) {
    TORCH_CHECK(fields.size() == 6 || fields.size() == 9, "bnpk: fields are (base, starts, lens) of 2 or 3 fields");
    TORCH_CHECK(luts.size() * 3 == fields.size(), "bnpk: one lut (or None) per field");
    std::vector<bnpk_field> out(3, bnpk_field{nullptr, 0, nullptr, nullptr, nullptr});
    for (size_t f = 0; f < luts.size(); ++f) {
        const Rows r = need_rows(fields[3 * f], fields[3 * f + 1], fields[3 * f + 2], luts[f], fields[0]);
        TORCH_CHECK(r.n_rows == (size_t)fields[2].numel(), "bnpk: fields differ in entry count");
        out[f] = bnpk_field{r.base, r.base_bytes, r.starts, r.lens, r.lut};
    }
    return out;
}

std::tuple<Tensor, Tensor> format_offsets(int64_t format, int64_t line_width, const std::vector<Tensor> &fields,
                                          const std::vector<c10::optional<Tensor>> &luts) {
    std::vector<bnpk_field> f = make_fields(fields, luts);
    c10::cuda::CUDAGuard guard(fields[0].device());
    const int64_t n = fields[2].numel();
    Tensor offsets = torch::empty({n + 1}, fields[0].options().dtype(torch::kInt64));
    Tensor status = new_status(fields[0]);
    Tensor ws = new_workspace(fields[0], (size_t)std::max<int64_t>(n, 1));
    check(bnpk_format_offsets((int)format, (int)line_width, (size_t)n, f.data(), offsets.data_ptr<int64_t>(),
                              status.data_ptr<int64_t>(), ws.data_ptr<uint8_t>(), (size_t)ws.numel(), cur_stream(fields[0])),
          "format_offsets");
    return {offsets, status};
}

Tensor format_records(int64_t format, int64_t line_width, const std::vector<Tensor> &fields,
                      const std::vector<c10::optional<Tensor>> &luts, const Tensor &offsets, int64_t out_begin,
                      int64_t out_end) {
    std::vector<bnpk_field> f = make_fields(fields, luts);
    const int64_t *offs = need_offsets(offsets, (size_t)fields[2].numel(), fields[0]);
    TORCH_CHECK(out_end >= out_begin, "bnpk: out_end < out_begin");
    c10::cuda::CUDAGuard guard(fields[0].device());
    Tensor out = torch::empty({out_end - out_begin}, fields[0].options().dtype(torch::kUInt8));
    check(bnpk_format_records((int)format, (int)line_width, (size_t)fields[2].numel(), f.data(),
                              offs, out_begin, out_end, out.numel() ? out.data_ptr<uint8_t>() : nullptr,
                              cur_stream(fields[0])),
          "format_records");
    return out;
}

// BED columns: per column of `kinds` (BNPK_COL_*) a value tensor (int64 text starts / int64 values / uint8 strand codes,
// empty for a skipped column) and a lens tensor (int32 for text, else empty); and the status block
std::tuple<std::vector<Tensor>, std::vector<Tensor>, Tensor> delimited_columns(const Tensor &chunk, const Tensor &starts,
                                                                               const Tensor &lens, c10::IntArrayRef kinds) {
    const Rows r = need_rows(chunk, starts, lens, c10::nullopt);
    TORCH_CHECK(!kinds.empty() && kinds.size() <= BNPK_MAX_COLUMNS, "bnpk: 1 to BNPK_MAX_COLUMNS columns");
    c10::cuda::CUDAGuard guard(chunk.device());
    const int64_t n = (int64_t)r.n_rows;
    std::vector<Tensor> values, text_lens;
    std::vector<bnpk_column> cols(kinds.size());
    for (size_t c = 0; c < kinds.size(); ++c) {
        const int64_t k = kinds[c];
        const bool named = k == BNPK_COL_TEXT || k == BNPK_COL_INT || k == BNPK_COL_INT_OR_DOT || k == BNPK_COL_STRAND;
        values.push_back(torch::empty({named ? n : 0}, chunk.options().dtype(k == BNPK_COL_STRAND ? torch::kUInt8 : torch::kInt64)));
        text_lens.push_back(torch::empty({k == BNPK_COL_TEXT ? n : 0}, chunk.options().dtype(torch::kInt32)));
        cols[c] = bnpk_column{(int)k, named ? values.back().data_ptr() : nullptr,
                              k == BNPK_COL_TEXT ? text_lens.back().data_ptr<int32_t>() : nullptr};
    }
    Tensor status = new_status(chunk);
    check(bnpk_delimited_columns(r.base, r.base_bytes, r.starts, r.lens, r.n_rows, cols.data(), (int)cols.size(),
                                 status.data_ptr<int64_t>(), cur_stream(chunk)),
          "delimited_columns");
    return {values, text_lens, status};
}

// contig index of every row's name in the sorted table (names, name_offsets int64[C+1]), -1 = unknown; and status
std::tuple<Tensor, Tensor> name_lookup(const Tensor &base, const Tensor &starts, const Tensor &lens, const Tensor &names,
                                       const Tensor &name_offsets) {
    const Rows r = need_rows(base, starts, lens, c10::nullopt);
    need(names, torch::kUInt8, "names", base);
    need(name_offsets, torch::kInt64, "name_offsets", base);
    TORCH_CHECK(name_offsets.numel() >= 1, "bnpk: name_offsets needs C + 1 entries");
    c10::cuda::CUDAGuard guard(base.device());
    Tensor ids = torch::empty({(int64_t)r.n_rows}, base.options().dtype(torch::kInt32));
    Tensor status = new_status(base);
    check(bnpk_name_lookup(r.base, r.base_bytes, r.starts, r.lens, r.n_rows, u8(names), name_offsets.data_ptr<int64_t>(),
                           (size_t)name_offsets.numel() - 1, ids.data_ptr<int32_t>(), status.data_ptr<int64_t>(),
                           cur_stream(base)),
          "name_lookup");
    return {ids, status};
}

// interval gather over a file image: ids (int32) index contigs = [offset int64, lenc int32, lenb int32, length int64];
// no ids = one flat contig.  check: (row_lens int32, status); copy: uint8[total] at offsets (int64[R+1])
struct Intervals {
    const int32_t *ids = nullptr;
    const int64_t *offset = nullptr, *length = nullptr;
    const int32_t *lenc = nullptr, *lenb = nullptr;
    size_t n_contigs = 0;
};
Intervals need_intervals(const Tensor &file, const Tensor &start, const Tensor &stop, const c10::optional<Tensor> &ids,
                         const std::vector<Tensor> &contigs) {
    need(file, torch::kUInt8, "file");
    need(start, torch::kInt64, "start", file);
    need(stop, torch::kInt64, "stop", file);
    TORCH_CHECK(start.numel() == stop.numel(), "bnpk: start and stop differ in length");
    Intervals iv;
    if (!ids) return iv;
    need(*ids, torch::kInt32, "ids", file);
    TORCH_CHECK(ids->numel() == start.numel(), "bnpk: one contig id per interval");
    TORCH_CHECK(contigs.size() == 4, "bnpk: contigs are [offset, lenc, lenb, length]");
    need(contigs[0], torch::kInt64, "contig_offset", file);
    need(contigs[1], torch::kInt32, "lenc", file);
    need(contigs[2], torch::kInt32, "lenb", file);
    need(contigs[3], torch::kInt64, "contig_len", file);
    const int64_t c = contigs[0].numel();
    TORCH_CHECK(contigs[1].numel() == c && contigs[2].numel() == c && contigs[3].numel() == c,
                "bnpk: the contig columns differ in length");
    iv.ids = ids->data_ptr<int32_t>();
    iv.offset = contigs[0].data_ptr<int64_t>();
    iv.lenc = contigs[1].data_ptr<int32_t>();
    iv.lenb = contigs[2].data_ptr<int32_t>();
    iv.length = contigs[3].data_ptr<int64_t>();
    iv.n_contigs = (size_t)c;
    return iv;
}

std::tuple<Tensor, Tensor> interval_check(const Tensor &file, const Tensor &start, const Tensor &stop,
                                          const c10::optional<Tensor> &ids, const std::vector<Tensor> &contigs) {
    const Intervals iv = need_intervals(file, start, stop, ids, contigs);
    c10::cuda::CUDAGuard guard(file.device());
    Tensor row_lens = torch::empty({start.numel()}, file.options().dtype(torch::kInt32));
    Tensor status = new_status(file);
    check(bnpk_interval_gather(u8(file), (size_t)file.numel(), (size_t)start.numel(), iv.ids, iv.offset, iv.lenc, iv.lenb,
                               iv.length, iv.n_contigs, start.data_ptr<int64_t>(), stop.data_ptr<int64_t>(), nullptr,
                               nullptr, row_lens.data_ptr<int32_t>(), nullptr, nullptr, status.data_ptr<int64_t>(),
                               cur_stream(file)),
          "interval_check");
    return {row_lens, status};
}

Tensor interval_copy(const Tensor &file, const Tensor &start, const Tensor &stop, const c10::optional<Tensor> &ids,
                     const std::vector<Tensor> &contigs, const c10::optional<Tensor> &strand,
                     const c10::optional<Tensor> &complement_lut, const Tensor &offsets, int64_t total) {
    const Intervals iv = need_intervals(file, start, stop, ids, contigs);
    const int64_t *offs = need_offsets(offsets, (size_t)start.numel(), file);
    const uint8_t *s = nullptr;
    if (strand) {
        need(*strand, torch::kUInt8, "strand", file);
        TORCH_CHECK(strand->numel() == start.numel(), "bnpk: one strand flag per interval");
        s = strand->data_ptr<uint8_t>();
    }
    const uint8_t *lut = need_lut(complement_lut, "complement_lut", file);
    c10::cuda::CUDAGuard guard(file.device());
    Tensor out = torch::empty({total}, file.options());
    if (total)
        check(bnpk_interval_gather(u8(file), (size_t)file.numel(), (size_t)start.numel(), iv.ids, iv.offset, iv.lenc,
                                   iv.lenb, iv.length, iv.n_contigs, start.data_ptr<int64_t>(), stop.data_ptr<int64_t>(),
                                   s, lut, nullptr, offs, out.data_ptr<uint8_t>(), nullptr, cur_stream(file)),
              "interval_copy");
    return out;
}

// pileups: event keys int64[2R] and the first bad row in the status block; ids (int32) index contig_offset and
// contig_len (int64), no ids = one contig of `size`
std::tuple<Tensor, Tensor> interval_events(const Tensor &start, const Tensor &stop, const c10::optional<Tensor> &ids,
                                           const c10::optional<Tensor> &contig_offset,
                                           const c10::optional<Tensor> &contig_len, int64_t size) {
    need(start, torch::kInt64, "start");
    need(stop, torch::kInt64, "stop", start);
    TORCH_CHECK(start.numel() == stop.numel(), "bnpk: start and stop differ in length");
    const int32_t *id = nullptr;
    const int64_t *off = nullptr, *len = nullptr;
    size_t n_contigs = 0;
    if (ids) {
        need(*ids, torch::kInt32, "ids", start);
        TORCH_CHECK(ids->numel() == start.numel(), "bnpk: one contig id per interval");
        TORCH_CHECK(contig_offset && contig_len, "bnpk: contig ids need contig_offset and contig_len");
        need(*contig_offset, torch::kInt64, "contig_offset", start);
        need(*contig_len, torch::kInt64, "contig_len", start);
        TORCH_CHECK(contig_offset->numel() == contig_len->numel(), "bnpk: the contig columns differ in length");
        id = ids->data_ptr<int32_t>();
        off = contig_offset->data_ptr<int64_t>();
        len = contig_len->data_ptr<int64_t>();
        n_contigs = (size_t)contig_offset->numel();
    }
    c10::cuda::CUDAGuard guard(start.device());
    Tensor keys = torch::empty({2 * start.numel()}, start.options());
    Tensor status = new_status(start);
    check(bnpk_interval_events(start.data_ptr<int64_t>(), stop.data_ptr<int64_t>(), id, off, len, n_contigs, size,
                               (size_t)start.numel(), keys.data_ptr<int64_t>(), nullptr, nullptr,
                               status.data_ptr<int64_t>(), cur_stream(start)),
          "interval_events");
    return {keys, status};
}

// runs of the coverage of sorted event keys: (run_starts int64[K + 2], run_values int64[K + 1], n_runs int64[1])
std::tuple<Tensor, Tensor, Tensor> pileup_runs(const Tensor &keys, int64_t size, int64_t mode) {
    need(keys, torch::kInt64, "keys");
    c10::cuda::CUDAGuard guard(keys.device());
    const int64_t n = keys.numel();
    Tensor starts = torch::empty({n + 2}, keys.options());
    Tensor values = torch::empty({n + 1}, keys.options());
    Tensor n_runs = torch::empty({1}, keys.options());
    Tensor ws = new_workspace(keys, (size_t)std::max<int64_t>(n, 1));
    check(bnpk_pileup_runs(n ? keys.data_ptr<int64_t>() : nullptr, (size_t)n, size, (int)mode,
                           starts.data_ptr<int64_t>(), values.data_ptr<int64_t>(), n_runs.data_ptr<int64_t>(),
                           ws.data_ptr<uint8_t>(), (size_t)ws.numel(), cur_stream(keys)),
          "pileup_runs");
    return {starts, values, n_runs};
}

// a track: run_starts int64[R + 1] and values int64[R]
void need_track(const Tensor &run_starts, const Tensor &values) {
    need(run_starts, torch::kInt64, "run_starts");
    need(values, torch::kInt64, "values", run_starts);
    TORCH_CHECK(values.numel() >= 1 && run_starts.numel() == values.numel() + 1,
                "bnpk: a track is R >= 1 values and R + 1 run starts");
}

Tensor runs_reduce(const Tensor &run_starts, const Tensor &values, const Tensor &q_start, const Tensor &q_stop,
                   int64_t mode) {
    need_track(run_starts, values);
    need(q_start, torch::kInt64, "q_start", run_starts);
    need(q_stop, torch::kInt64, "q_stop", run_starts);
    TORCH_CHECK(q_start.numel() == q_stop.numel(), "bnpk: q_start and q_stop differ in length");
    c10::cuda::CUDAGuard guard(run_starts.device());
    const int64_t n = q_start.numel();
    Tensor out = torch::empty({n}, run_starts.options());
    Tensor scratch = torch::empty({3 * n + 1}, run_starts.options());
    Tensor ws = new_workspace(run_starts, (size_t)std::max<int64_t>(n, 1));
    check(bnpk_runs_reduce(run_starts.data_ptr<int64_t>(), values.data_ptr<int64_t>(), (size_t)values.numel(),
                           q_start.data_ptr<int64_t>(), q_stop.data_ptr<int64_t>(), (size_t)n, (int)mode,
                           out.data_ptr<int64_t>(), scratch.data_ptr<int64_t>(), ws.data_ptr<uint8_t>(),
                           (size_t)ws.numel(), cur_stream(run_starts)),
          "runs_reduce");
    return out;
}

Tensor runs_extract(const Tensor &run_starts, const Tensor &values, const Tensor &q_start, const Tensor &offsets,
                    int64_t total) {
    need_track(run_starts, values);
    need(q_start, torch::kInt64, "q_start", run_starts);
    const int64_t *offs = need_offsets(offsets, (size_t)q_start.numel(), run_starts);
    c10::cuda::CUDAGuard guard(run_starts.device());
    Tensor out = torch::empty({total}, run_starts.options());
    if (total)
        check(bnpk_runs_extract(run_starts.data_ptr<int64_t>(), values.data_ptr<int64_t>(), (size_t)values.numel(),
                                q_start.data_ptr<int64_t>(), (size_t)q_start.numel(), offs, out.data_ptr<int64_t>(),
                                cur_stream(run_starts)),
              "runs_extract");
    return out;
}

// merge: (out_rows int64[R], out_stops int64[R], n_out int64[1], status)
std::tuple<Tensor, Tensor, Tensor, Tensor> interval_merge(const Tensor &start, const Tensor &stop,
                                                          const c10::optional<Tensor> &same_prev, int64_t distance) {
    need(start, torch::kInt64, "start");
    need(stop, torch::kInt64, "stop", start);
    TORCH_CHECK(start.numel() == stop.numel(), "bnpk: start and stop differ in length");
    const uint8_t *sp = nullptr;
    if (same_prev) {
        need(*same_prev, torch::kUInt8, "same_prev", start);
        TORCH_CHECK(same_prev->numel() == start.numel(), "bnpk: one same_prev flag per row");
        sp = u8(*same_prev);
    }
    c10::cuda::CUDAGuard guard(start.device());
    const int64_t n = start.numel();
    Tensor rows = torch::empty({n}, start.options());
    Tensor stops = torch::empty({n}, start.options());
    Tensor n_out = torch::empty({1}, start.options());
    Tensor status = new_status(start);
    Tensor ws = new_workspace(start, (size_t)std::max<int64_t>(n, 1));
    check(bnpk_interval_merge(start.data_ptr<int64_t>(), stop.data_ptr<int64_t>(), sp, (size_t)n, distance,
                              rows.data_ptr<int64_t>(), stops.data_ptr<int64_t>(), n_out.data_ptr<int64_t>(),
                              status.data_ptr<int64_t>(), ws.data_ptr<uint8_t>(), (size_t)ws.numel(), cur_stream(start)),
          "interval_merge");
    return {rows, stops, n_out, status};
}

Tensor rows_equal_prev(const Tensor &base, const Tensor &starts, const Tensor &lens) {
    const Rows r = need_rows(base, starts, lens, c10::nullopt);
    c10::cuda::CUDAGuard guard(base.device());
    Tensor flag = torch::empty({(int64_t)r.n_rows}, base.options());
    check(r.call(bnpk_rows_equal_prev, flag.data_ptr<uint8_t>(), cur_stream(base)), "rows_equal_prev");
    return flag;
}

// op(A, B) of two tracks: (run_starts int64[Ra + Rb + 1], run_values int64[max(Ra + Rb, 1)], n_runs int64[1])
std::tuple<Tensor, Tensor, Tensor> runs_combine(const Tensor &a_starts, const Tensor &a_values, const Tensor &b_starts,
                                                const Tensor &b_values, int64_t op) {
    need(a_starts, torch::kInt64, "a_starts");
    need(a_values, torch::kInt64, "a_values", a_starts);
    need(b_starts, torch::kInt64, "b_starts", a_starts);
    need(b_values, torch::kInt64, "b_values", a_starts);
    TORCH_CHECK(a_starts.numel() == a_values.numel() + 1 && b_starts.numel() == b_values.numel() + 1,
                "bnpk: a track is R values and R + 1 run starts");
    c10::cuda::CUDAGuard guard(a_starts.device());
    const int64_t n = a_values.numel() + b_values.numel();
    Tensor starts = torch::empty({n + 1}, a_starts.options());
    Tensor values = torch::empty({std::max<int64_t>(n, 1)}, a_starts.options());
    Tensor n_runs = torch::empty({1}, a_starts.options());
    Tensor ws = new_workspace(a_starts, (size_t)std::max<int64_t>(n, 1));
    check(bnpk_runs_combine(a_starts.data_ptr<int64_t>(), a_values.data_ptr<int64_t>(), (size_t)a_values.numel(),
                            b_starts.data_ptr<int64_t>(), b_values.data_ptr<int64_t>(), (size_t)b_values.numel(),
                            (int)op, starts.data_ptr<int64_t>(), values.data_ptr<int64_t>(), n_runs.data_ptr<int64_t>(),
                            ws.data_ptr<uint8_t>(), (size_t)ws.numel(), cur_stream(a_starts)),
          "runs_combine");
    return {starts, values, n_runs};
}

// intersect: (out_rows int64[R], out_stops int64[R], n_out int64[1], overlap int64[1]); rows=False leaves the first
// two empty and counts only
std::tuple<Tensor, Tensor, Tensor, Tensor> interval_intersect(const Tensor &start, const Tensor &stop,
                                                              const c10::optional<Tensor> &same_prev, bool rows) {
    need(start, torch::kInt64, "start");
    need(stop, torch::kInt64, "stop", start);
    TORCH_CHECK(start.numel() == stop.numel(), "bnpk: start and stop differ in length");
    const uint8_t *sp = nullptr;
    if (same_prev) {
        need(*same_prev, torch::kUInt8, "same_prev", start);
        TORCH_CHECK(same_prev->numel() == start.numel(), "bnpk: one same_prev flag per row");
        sp = u8(*same_prev);
    }
    c10::cuda::CUDAGuard guard(start.device());
    const int64_t n = start.numel();
    Tensor out_rows = torch::empty({rows ? n : 0}, start.options());
    Tensor out_stops = torch::empty({rows ? n : 0}, start.options());
    Tensor n_out = torch::empty({1}, start.options());
    Tensor overlap = torch::empty({1}, start.options());
    Tensor ws = new_workspace(start, (size_t)std::max<int64_t>(n, 1));
    check(bnpk_interval_intersect(start.data_ptr<int64_t>(), stop.data_ptr<int64_t>(), sp, (size_t)n,
                                  rows ? out_rows.data_ptr<int64_t>() : nullptr,
                                  rows ? out_stops.data_ptr<int64_t>() : nullptr, n_out.data_ptr<int64_t>(),
                                  overlap.data_ptr<int64_t>(), ws.data_ptr<uint8_t>(), (size_t)ws.numel(),
                                  cur_stream(start)),
          "interval_intersect");
    return {out_rows, out_stops, n_out, overlap};
}

// a track's rows: (contig int32[R + C], start, stop, value int64[R + C], n_out int64[1]), the first n_out valid
std::tuple<Tensor, Tensor, Tensor, Tensor, Tensor> runs_to_intervals(const Tensor &run_starts, const Tensor &values,
                                                                     const Tensor &contig_ends, int64_t mode) {
    need(run_starts, torch::kInt64, "run_starts");
    need(values, torch::kInt64, "values", run_starts);
    need(contig_ends, torch::kInt64, "contig_ends", run_starts);
    TORCH_CHECK(run_starts.numel() == values.numel() + 1, "bnpk: a track is R values and R + 1 run starts");
    TORCH_CHECK(contig_ends.numel() >= 2, "bnpk: contig_ends holds 0 and the end of every contig");
    c10::cuda::CUDAGuard guard(run_starts.device());
    const int64_t n = values.numel(), c = contig_ends.numel() - 1;
    Tensor contig = torch::empty({n + c}, run_starts.options().dtype(torch::kInt32));
    Tensor start = torch::empty({n + c}, run_starts.options());
    Tensor stop = torch::empty({n + c}, run_starts.options());
    Tensor value = torch::empty({n + c}, run_starts.options());
    Tensor n_out = torch::empty({1}, run_starts.options());
    Tensor ws = new_workspace(run_starts, (size_t)std::max<int64_t>(n, 1));
    check(bnpk_runs_to_intervals(run_starts.data_ptr<int64_t>(), values.data_ptr<int64_t>(), (size_t)n,
                                 contig_ends.data_ptr<int64_t>(), (size_t)c, (int)mode, contig.data_ptr<int32_t>(),
                                 start.data_ptr<int64_t>(), stop.data_ptr<int64_t>(), value.data_ptr<int64_t>(),
                                 n_out.data_ptr<int64_t>(), ws.data_ptr<uint8_t>(), (size_t)ws.numel(),
                                 cur_stream(run_starts)),
          "runs_to_intervals");
    return {contig, start, stop, value, n_out};
}

// delimited columns: `kinds` names each column's kind; a TEXT column takes three tensors of `columns` (base uint8,
// starts int64, lens int32), an INT column one int64 and a STRAND column one uint8 tensor, each with one row per line
struct OutColumns {
    bnpk_out_column col[BNPK_MAX_OUT_COLUMNS];
    int n_cols;
    size_t n_lines;
};

OutColumns need_out_columns(const std::vector<Tensor> &columns, const std::vector<int64_t> &kinds) {
    TORCH_CHECK(!kinds.empty() && kinds.size() <= BNPK_MAX_OUT_COLUMNS, "bnpk: 1 to 8 columns");
    OutColumns oc{};
    oc.n_cols = (int)kinds.size();
    size_t t = 0;
    int64_t rows = -1;
    for (size_t k = 0; k < kinds.size(); ++k) {
        bnpk_out_column &c = oc.col[k];
        c.kind = (int)kinds[k];
        int64_t n = 0;
        if (c.kind == BNPK_COL_TEXT) {
            TORCH_CHECK(t + 3 <= columns.size(), "bnpk: a text column is three tensors");
            const Rows r = need_rows(columns[t], columns[t + 1], columns[t + 2], c10::nullopt, columns[0]);
            c.data = r.base;
            c.base_bytes = r.base_bytes;
            c.starts = r.starts;
            c.lens = r.lens;
            n = (int64_t)r.n_rows;
            t += 3;
        } else {
            TORCH_CHECK(c.kind == BNPK_COL_INT || c.kind == BNPK_COL_STRAND, "bnpk: a column is TEXT, INT or STRAND");
            TORCH_CHECK(t < columns.size(), "bnpk: a column misses its tensor");
            need(columns[t], c.kind == BNPK_COL_INT ? torch::kInt64 : torch::kUInt8, "column", columns[0]);
            c.data = columns[t].data_ptr();
            n = columns[t].numel();
            t += 1;
        }
        TORCH_CHECK(rows < 0 || n == rows, "bnpk: the columns differ in length");
        rows = n;
    }
    TORCH_CHECK(t == columns.size(), "bnpk: more tensors than the kinds name");
    oc.n_lines = (size_t)rows;
    return oc;
}

std::tuple<Tensor, Tensor> delimited_offsets(const std::vector<Tensor> &columns, const std::vector<int64_t> &kinds) {
    const OutColumns oc = need_out_columns(columns, kinds);
    const Tensor &like = columns[0];
    c10::cuda::CUDAGuard guard(like.device());
    Tensor offsets = torch::empty({(int64_t)oc.n_lines + 1}, like.options().dtype(torch::kInt64));
    Tensor status = new_status(like);
    Tensor ws = new_workspace(like, std::max<size_t>(oc.n_lines, 1));
    check(bnpk_delimited_offsets(oc.col, oc.n_cols, oc.n_lines, offsets.data_ptr<int64_t>(), status.data_ptr<int64_t>(),
                                 ws.data_ptr<uint8_t>(), (size_t)ws.numel(), cur_stream(like)),
          "delimited_offsets");
    return {offsets, status};
}

Tensor delimited_format(const std::vector<Tensor> &columns, const std::vector<int64_t> &kinds, const Tensor &offsets,
                        int64_t out_begin, int64_t out_end) {
    const OutColumns oc = need_out_columns(columns, kinds);
    const int64_t *offs = need_offsets(offsets, oc.n_lines, columns[0]);
    TORCH_CHECK(0 <= out_begin && out_begin <= out_end, "bnpk: need 0 <= out_begin <= out_end");
    c10::cuda::CUDAGuard guard(offsets.device());
    Tensor out = torch::empty({out_end - out_begin}, offsets.options().dtype(torch::kUInt8));
    if (out_end > out_begin)
        check(bnpk_delimited_format(oc.col, oc.n_cols, oc.n_lines, offs, out_begin, out_end, out.data_ptr<uint8_t>(),
                                    cur_stream(offsets)),
              "delimited_format");
    return out;
}

// BAM records: (starts int64[n / 36 + 1], status); the first status[N_RECORDS] starts are the complete records
std::tuple<Tensor, Tensor> bam_split(const Tensor &chunk, int64_t n_ref, int64_t segment_bytes) {
    need(chunk, torch::kUInt8, "chunk");
    TORCH_CHECK(segment_bytes >= 64, "bnpk: segment_bytes must be at least 64");
    c10::cuda::CUDAGuard guard(chunk.device());
    const int64_t n = chunk.numel();
    Tensor starts = torch::empty({n / 36 + 1}, chunk.options().dtype(torch::kInt64));
    Tensor status = new_status(chunk);
    Tensor ws = torch::empty({7 * std::max<int64_t>((n + segment_bytes - 1) / segment_bytes, 1)}, starts.options());
    check(bnpk_bam_split(u8(chunk), (size_t)n, (int)n_ref, (size_t)segment_bytes, starts.data_ptr<int64_t>(),
                         (size_t)starts.numel(), status.data_ptr<int64_t>(), ws.data_ptr<int64_t>(), (size_t)ws.numel(),
                         cur_stream(chunk)),
          "bam_split");
    return {starts, status};
}

// the fields of the records bam_split found: int64[BNPK_BAM_FIELDS, starts.numel()]
Tensor bam_fields(const Tensor &chunk, const Tensor &starts, Tensor status) {
    need(chunk, torch::kUInt8, "chunk");
    need(starts, torch::kInt64, "starts", chunk);
    need(status, torch::kInt64, "status", chunk);
    TORCH_CHECK(status.numel() >= BNPK_ST_WORDS, "bnpk: status must have BNPK_ST_WORDS words");
    c10::cuda::CUDAGuard guard(chunk.device());
    Tensor fields = torch::empty({BNPK_BAM_FIELDS, starts.numel()}, starts.options());
    check(bnpk_bam_fields(u8(chunk), (size_t)chunk.numel(), starts.data_ptr<int64_t>(), (size_t)starts.numel(),
                          fields.data_ptr<int64_t>(), status.data_ptr<int64_t>(), cur_stream(chunk)),
          "bam_fields");
    return fields;
}

Tensor bam_sequence(const Tensor &chunk, const Tensor &seq_start, const Tensor &offsets, int64_t total) {
    need(chunk, torch::kUInt8, "chunk");
    need(seq_start, torch::kInt64, "seq_start", chunk);
    const int64_t *off = need_offsets(offsets, (size_t)seq_start.numel(), chunk);
    c10::cuda::CUDAGuard guard(chunk.device());
    Tensor out = torch::empty({total}, chunk.options());
    if (total == 0) return out;
    check(bnpk_bam_sequence(u8(chunk), (size_t)chunk.numel(), seq_start.data_ptr<int64_t>(), off,
                            (size_t)seq_start.numel(), out.data_ptr<uint8_t>(), cur_stream(chunk)),
          "bam_sequence");
    return out;
}

std::tuple<Tensor, Tensor> bam_cigar(const Tensor &chunk, const Tensor &cigar_start, const Tensor &offsets,
                                     int64_t total) {
    need(chunk, torch::kUInt8, "chunk");
    need(cigar_start, torch::kInt64, "cigar_start", chunk);
    const int64_t *off = need_offsets(offsets, (size_t)cigar_start.numel(), chunk);
    c10::cuda::CUDAGuard guard(chunk.device());
    Tensor op = torch::empty({total}, chunk.options());
    Tensor length = torch::empty({total}, cigar_start.options());
    if (total == 0) return {op, length};
    check(bnpk_bam_cigar(u8(chunk), (size_t)chunk.numel(), cigar_start.data_ptr<int64_t>(), off,
                         (size_t)cigar_start.numel(), op.data_ptr<uint8_t>(), length.data_ptr<int64_t>(),
                         cur_stream(chunk)),
          "bam_cigar");
    return {op, length};
}

}  // namespace

TORCH_LIBRARY(bnpk, m) {
    m.def("chunk_kmer_count(Tensor chunk, int k, int window_size, Tensor(a!) hist, int lines_per_entry=4, "
          "int header_char=64, bool check_plus=True, int trim_cr=-1, int enc_mode=0, Tensor? lut=None, "
          "int hist_mode=0) -> Tensor");
    m.def("line_split(Tensor chunk, int lines_per_entry, int field_line, int start_offset, int header_char, "
          "bool check_plus, int trim_cr, int max_rows) -> (Tensor, Tensor, Tensor)");
    m.def("row_offsets(Tensor lens, int shrink) -> Tensor");
    m.def("rows_encode(Tensor base, Tensor starts, Tensor lens, int enc_mode, Tensor? lut, Tensor offsets, int total) "
          "-> (Tensor, Tensor)");
    m.def("rows_kmer_hash(Tensor base, Tensor starts, Tensor lens, int enc_mode, Tensor? lut, int k, int window_size, "
          "int complement_xor, Tensor offsets, int total) -> (Tensor, Tensor)");
    m.def("rows_kmer_count(Tensor base, Tensor starts, Tensor lens, int enc_mode, Tensor? lut, int k, int window_size, "
          "int complement_xor, Tensor(a!) hist, int hist_mode=0) -> Tensor");
    m.def("rows_kmer_table_insert(Tensor base, Tensor starts, Tensor lens, int enc_mode, Tensor? lut, int k, "
          "int complement_xor, Tensor(a!) keys, Tensor(b!) counts, Tensor(c!) n_used) -> Tensor");
    m.def("rows_reverse_complement(Tensor base, Tensor starts, Tensor lens, Tensor lut, Tensor offsets, int total) -> Tensor");
    m.def("rows_pwm_scores(Tensor base, Tensor starts, Tensor lens, int enc_mode, Tensor? lut, Tensor matrix, bool tail, "
          "Tensor offsets, int total) -> (Tensor, Tensor)");
    m.def("rows_match(Tensor base, Tensor starts, Tensor lens, int enc_mode, Tensor? lut, int alphabet_size, Tensor sets, "
          "int[] sub_lens, bool same, Tensor offsets, int total) -> (Tensor, Tensor)");
    m.def("bincount(Tensor values, Tensor(a!) hist, int hist_mode=0) -> Tensor");
    m.def("format_offsets(int format, int line_width, Tensor[] fields, Tensor?[] luts) -> (Tensor, Tensor)");
    m.def("format_records(int format, int line_width, Tensor[] fields, Tensor?[] luts, Tensor offsets, int out_begin, "
          "int out_end) -> Tensor");
    m.def("delimited_columns(Tensor chunk, Tensor starts, Tensor lens, int[] kinds) -> (Tensor[], Tensor[], Tensor)");
    m.def("name_lookup(Tensor base, Tensor starts, Tensor lens, Tensor names, Tensor name_offsets) -> (Tensor, Tensor)");
    m.def("interval_check(Tensor file, Tensor start, Tensor stop, Tensor? ids, Tensor[] contigs) -> (Tensor, Tensor)");
    m.def("interval_copy(Tensor file, Tensor start, Tensor stop, Tensor? ids, Tensor[] contigs, Tensor? strand, "
          "Tensor? complement_lut, Tensor offsets, int total) -> Tensor");
    m.def("interval_events(Tensor start, Tensor stop, Tensor? ids, Tensor? contig_offset, Tensor? contig_len, int size) "
          "-> (Tensor, Tensor)");
    m.def("pileup_runs(Tensor keys, int size, int mode) -> (Tensor, Tensor, Tensor)");
    m.def("runs_reduce(Tensor run_starts, Tensor values, Tensor q_start, Tensor q_stop, int mode) -> Tensor");
    m.def("runs_extract(Tensor run_starts, Tensor values, Tensor q_start, Tensor offsets, int total) -> Tensor");
    m.def("interval_merge(Tensor start, Tensor stop, Tensor? same_prev, int distance) -> (Tensor, Tensor, Tensor, Tensor)");
    m.def("rows_equal_prev(Tensor base, Tensor starts, Tensor lens) -> Tensor");
    m.def("runs_combine(Tensor a_starts, Tensor a_values, Tensor b_starts, Tensor b_values, int op) "
          "-> (Tensor, Tensor, Tensor)");
    m.def("interval_intersect(Tensor start, Tensor stop, Tensor? same_prev, bool rows) "
          "-> (Tensor, Tensor, Tensor, Tensor)");
    m.def("runs_to_intervals(Tensor run_starts, Tensor values, Tensor contig_ends, int mode) "
          "-> (Tensor, Tensor, Tensor, Tensor, Tensor)");
    m.def("delimited_offsets(Tensor[] columns, int[] kinds) -> (Tensor, Tensor)");
    m.def("delimited_format(Tensor[] columns, int[] kinds, Tensor offsets, int out_begin, int out_end) -> Tensor");
    m.def("bam_split(Tensor chunk, int n_ref, int segment_bytes=4096) -> (Tensor, Tensor)");
    m.def("bam_fields(Tensor chunk, Tensor starts, Tensor(a!) status) -> Tensor");
    m.def("bam_sequence(Tensor chunk, Tensor seq_start, Tensor offsets, int total) -> Tensor");
    m.def("bam_cigar(Tensor chunk, Tensor cigar_start, Tensor offsets, int total) -> (Tensor, Tensor)");
}

TORCH_LIBRARY_IMPL(bnpk, CUDA, m) {
    m.impl("chunk_kmer_count", &chunk_kmer_count);
    m.impl("line_split", &line_split);
    m.impl("row_offsets", &row_offsets);
    m.impl("rows_encode", &rows_encode);
    m.impl("rows_kmer_hash", &rows_kmer_hash);
    m.impl("rows_kmer_count", &rows_kmer_count);
    m.impl("rows_kmer_table_insert", &rows_kmer_table_insert);
    m.impl("rows_reverse_complement", &rows_reverse_complement);
    m.impl("rows_pwm_scores", &rows_pwm_scores);
    m.impl("rows_match", &rows_match);
    m.impl("bincount", &bincount);
    m.impl("format_offsets", &format_offsets);
    m.impl("format_records", &format_records);
    m.impl("delimited_columns", &delimited_columns);
    m.impl("name_lookup", &name_lookup);
    m.impl("interval_check", &interval_check);
    m.impl("interval_copy", &interval_copy);
    m.impl("interval_events", &interval_events);
    m.impl("pileup_runs", &pileup_runs);
    m.impl("runs_reduce", &runs_reduce);
    m.impl("runs_extract", &runs_extract);
    m.impl("interval_merge", &interval_merge);
    m.impl("rows_equal_prev", &rows_equal_prev);
    m.impl("runs_combine", &runs_combine);
    m.impl("interval_intersect", &interval_intersect);
    m.impl("runs_to_intervals", &runs_to_intervals);
    m.impl("delimited_offsets", &delimited_offsets);
    m.impl("delimited_format", &delimited_format);
    m.impl("bam_split", &bam_split);
    m.impl("bam_fields", &bam_fields);
    m.impl("bam_sequence", &bam_sequence);
    m.impl("bam_cigar", &bam_cigar);
}
