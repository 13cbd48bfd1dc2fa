"""ctypes binding of libbnpk.so (the C-ABI declared in include/bnpk.h).

There is NO fallback: if the CUDA library is missing or no CUDA device is present, every
compute entry point raises.  The oracle under ``oracle/`` is test infrastructure and is never
imported from here.
"""
import ctypes
import os

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "_lib", "libbnpk.so")

# mirror of include/bnpk.h -----------------------------------------------------------------
ENC_ASCII_ACGT, ENC_ASCII_ACTG, ENC_CODES, ENC_LUT = 0, 1, 2, 3
HIST_AUTO, HIST_SMEM, HIST_GLOBAL = 0, 1, 2
E_BADARG, E_K, E_WINDOW, E_WORKSPACE, E_BINS = -1, -2, -3, -4, -5
(ST_N_LINES, ST_N_RECORDS, ST_N_COMPLETE_BYTES, ST_BAD_HEADER_ENTRY, ST_BAD_PLUS_ENTRY, ST_BAD_BASE,
 ST_N_BASES, ST_N_VALUES, ST_N_LONG_ROWS, ST_CR, ST_LAST_ROW_START, ST_LAST_ROW_INDEX, ST_OVERFLOW,
 ST_TABLE_FULL) = range(14)
ST_WORDS = 16
FMT_FASTQ, FMT_FASTA, FMT_FASTA_WRAPPED = 0, 1, 2
MAX_COLUMNS = 16
COL_SKIP, COL_TEXT, COL_INT, COL_INT_OR_DOT, COL_STRAND = 0, 1, 2, 3, 4
BAD_TABS, BAD_COLUMNS, BAD_INT, BAD_STRAND = 1, 2, 3, 4
PILEUP_COUNT, PILEUP_ANY = 0, 1
RUNS_MAX, RUNS_MIN, RUNS_SUM, RUNS_ANY = 0, 1, 2, 3
(OP_ADD, OP_SUB, OP_MUL, OP_AND, OP_OR, OP_XOR, OP_MIN, OP_MAX, OP_EQ, OP_NE, OP_LT, OP_LE, OP_GT,
 OP_GE) = range(14)
RUNS_TO_NONZERO, RUNS_TO_ALL = 0, 1
MAX_OUT_COLUMNS = 8
BAM_BAD_BLOCK_SIZE, BAM_BAD_REF_ID, BAM_BAD_NAME, BAM_BAD_SIZES, BAM_BAD_CIGAR_OP, BAM_TRUNCATED = 1, 2, 3, 4, 5, 6
(BAM_F_REF_ID, BAM_F_POS, BAM_F_MAPQ, BAM_F_FLAG, BAM_F_NAME_START, BAM_F_NAME_LEN, BAM_F_CIGAR_START, BAM_F_N_CIGAR,
 BAM_F_SEQ_START, BAM_F_L_SEQ, BAM_F_QUAL_START, BAM_F_REF_LEN) = range(12)
BAM_FIELDS = 12
INT64_MAX = (1 << 63) - 1
SMEM_MAX_BINS = 32768

_vp, _sz, _i, _i64, _u8, _u64 = (ctypes.c_void_p, ctypes.c_size_t, ctypes.c_int, ctypes.c_int64,
                                 ctypes.c_uint8, ctypes.c_uint64)

# name -> (restype, argtypes); tests check every one of these is exported
SIGNATURES = {
    "bnpk_abi_version": (_i, []),
    "bnpk_last_error": (ctypes.c_char_p, []),
    "bnpk_sm_count": (_i, []),
    "bnpk_launch_count": (_u64, []),
    "bnpk_profile_enable": (_i, [_i]),
    "bnpk_profile_read": (_i, [ctypes.POINTER(ctypes.c_double), ctypes.POINTER(_u64)]),
    "bnpk_status_init": (_i, [_vp, _vp]),
    "bnpk_count_byte": (_i, [_vp, _sz, _u8, _vp, _vp]),
    "bnpk_tile_workspace_bytes": (_sz, [_sz]),
    "bnpk_tile_workspace_reset": (_i, [_vp, _sz, _vp]),
    "bnpk_line_split": (_i, [_vp, _sz, _i, _i, _i, _u8, _i, _i, _vp, _vp, _sz, _vp, _vp, _sz, _vp]),
    "bnpk_chunk_kmer_count": (_i, [_vp, _sz, _sz, _sz, _i, _i, _u8, _i, _i, _i, _vp, _i, _i, _i64, _i, _vp,
                                   _vp, _vp, _sz, _vp]),
    "bnpk_row_offsets": (_i, [_vp, _sz, _i, _vp, _vp, _sz, _vp]),
    "bnpk_rows_encode": (_i, [_vp, _sz, _vp, _vp, _sz, _i, _vp, _vp, _vp, _vp, _vp]),
    "bnpk_rows_kmer_hash": (_i, [_vp, _sz, _vp, _vp, _sz, _i, _vp, _i, _vp, _vp, _vp, _vp]),
    "bnpk_rows_generic_hash": (_i, [_vp, _sz, _vp, _vp, _sz, _vp, _i, _i, _vp, _vp, _vp, _vp]),
    "bnpk_rows_minimizers": (_i, [_vp, _sz, _vp, _vp, _sz, _i, _vp, _i, _i, _vp, _vp, _vp, _vp]),
    "bnpk_rows_kmer_count": (_i, [_vp, _sz, _vp, _vp, _sz, _i, _vp, _i, _i, _i64, _i, _vp, _vp, _vp]),
    "bnpk_rows_reverse_complement": (_i, [_vp, _sz, _vp, _vp, _sz, _vp, _vp, _vp, _vp]),
    "bnpk_rows_kmer_hash_canonical": (_i, [_vp, _sz, _vp, _vp, _sz, _i, _vp, _i, _i, _vp, _vp, _vp, _vp]),
    "bnpk_rows_kmer_count_canonical": (_i, [_vp, _sz, _vp, _vp, _sz, _i, _vp, _i, _i, _i64, _i, _vp, _vp, _vp]),
    "bnpk_rows_kmer_table_insert": (_i, [_vp, _sz, _vp, _vp, _sz, _i, _vp, _i, _i, _vp, _vp, _sz, _vp, _vp, _vp]),
    "bnpk_kmer_table_rehash": (_i, [_vp, _vp, _sz, _vp, _vp, _sz, _vp, _vp, _vp]),
    "bnpk_rows_pwm_scores": (_i, [_vp, _sz, _vp, _vp, _sz, _i, _vp, _i, _vp, _i, _i, _vp, _vp, _vp, _vp]),
    "bnpk_rows_pwm_max": (_i, [_vp, _sz, _vp, _vp, _sz, _i, _vp, _i, _vp, _i, _vp, _vp, _vp]),
    "bnpk_rows_match": (_i, [_vp, _sz, _vp, _vp, _sz, _i, _vp, _i, _vp, _vp, _i, _i, _vp, _vp, _vp, _vp]),
    "bnpk_rows_match_count": (_i, [_vp, _sz, _vp, _vp, _sz, _i, _vp, _i, _vp, _vp, _i, _i, _vp, _vp, _vp]),
    "bnpk_bincount": (_i, [_vp, _sz, _i64, _i, _vp, _vp, _vp]),
    "bnpk_bincount_rows": (_i, [_vp, _vp, _sz, _i64, _vp, _vp, _vp]),
    "bnpk_pipeline_create": (_i, [ctypes.POINTER(_vp), _sz, _sz]),
    "bnpk_pipeline_destroy": (None, [_vp]),
    "bnpk_pipeline_kmer_count_host": (_i, [_vp, _vp, _sz, _i, _u8, _i, _i, _i, _vp, _i, _i, _i64, _i, _vp, _vp]),
    "bnpk_pipeline_kmer_count_host_on": (_i, [_vp, _vp, _sz, _i, _u8, _i, _i, _i, _vp, _i, _i, _i64, _i, _vp, _vp, _vp]),
    "bnpk_multiline_flags": (_i, [_vp, _sz, _vp, _vp, _sz, _vp, _vp, _vp]),
    "bnpk_multiline_entries": (_i, [_vp, _vp, _vp, _vp, _vp, _sz, _i, _vp, _vp, _vp, _vp, _vp, _vp]),
    "bnpk_bloom_insert": (_i, [_vp, _sz, _vp, _i, _vp, _sz, _vp]),
    "bnpk_bloom_query": (_i, [_vp, _sz, _vp, _i, _vp, _sz, _vp, _vp]),
    "bnpk_synth_fastq": (_i, [_vp, _u64, _u64, _u64, _vp]),
    "bnpk_format_offsets": (_i, [_i, _i, _sz, _vp, _vp, _vp, _vp, _sz, _vp]),
    "bnpk_format_records": (_i, [_i, _i, _sz, _vp, _vp, _i64, _i64, _vp, _vp]),
    "bnpk_delimited_columns": (_i, [_vp, _sz, _vp, _vp, _sz, _vp, _i, _vp, _vp]),
    "bnpk_name_lookup": (_i, [_vp, _sz, _vp, _vp, _sz, _vp, _vp, _sz, _vp, _vp, _vp]),
    "bnpk_interval_gather": (_i, [_vp, _sz, _sz, _vp, _vp, _vp, _vp, _vp, _sz, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp,
                                  _vp]),
    "bnpk_interval_events": (_i, [_vp, _vp, _vp, _vp, _vp, _sz, _i64, _sz, _vp, _vp, _vp, _vp, _vp]),
    "bnpk_pileup_runs": (_i, [_vp, _sz, _i64, _i, _vp, _vp, _vp, _vp, _sz, _vp]),
    "bnpk_runs_reduce": (_i, [_vp, _vp, _sz, _vp, _vp, _sz, _i, _vp, _vp, _vp, _sz, _vp]),
    "bnpk_runs_extract": (_i, [_vp, _vp, _sz, _vp, _sz, _vp, _vp, _vp]),
    "bnpk_interval_merge": (_i, [_vp, _vp, _vp, _sz, _i64, _vp, _vp, _vp, _vp, _vp, _sz, _vp]),
    "bnpk_rows_equal_prev": (_i, [_vp, _sz, _vp, _vp, _sz, _vp, _vp]),
    "bnpk_runs_combine": (_i, [_vp, _vp, _sz, _vp, _vp, _sz, _i, _vp, _vp, _vp, _vp, _sz, _vp]),
    "bnpk_interval_intersect": (_i, [_vp, _vp, _vp, _sz, _vp, _vp, _vp, _vp, _vp, _sz, _vp]),
    "bnpk_runs_to_intervals": (_i, [_vp, _vp, _sz, _vp, _sz, _i, _vp, _vp, _vp, _vp, _vp, _vp, _sz, _vp]),
    "bnpk_delimited_offsets": (_i, [_vp, _i, _sz, _vp, _vp, _vp, _sz, _vp]),
    "bnpk_delimited_format": (_i, [_vp, _i, _sz, _vp, _i64, _i64, _vp, _vp]),
    "bnpk_bam_split": (_i, [_vp, _sz, _i, _sz, _vp, _sz, _vp, _vp, _sz, _vp]),
    "bnpk_bam_fields": (_i, [_vp, _sz, _vp, _sz, _vp, _vp, _vp]),
    "bnpk_bam_sequence": (_i, [_vp, _sz, _vp, _vp, _sz, _vp, _vp]),
    "bnpk_bam_cigar": (_i, [_vp, _sz, _vp, _vp, _sz, _vp, _vp, _vp]),
}


class Field(ctypes.Structure):
    """bnpk_field: a ragged view (base, starts, lens) and an optional device LUT applied on the way out."""
    _fields_ = [("base", _vp), ("base_bytes", _sz), ("starts", _vp), ("lens", _vp), ("lut256", _vp)]


class Column(ctypes.Structure):
    """bnpk_column: how one tab-separated column is written (COL_*), its output and, for text, its lengths."""
    _fields_ = [("kind", _i), ("out", _vp), ("lens", _vp)]


class OutColumn(ctypes.Structure):
    """bnpk_out_column: one written column (COL_TEXT, COL_INT or COL_STRAND), its data and, for text, its rows."""
    _fields_ = [("kind", _i), ("data", _vp), ("base_bytes", _sz), ("starts", _vp), ("lens", _vp)]


class NativeLibraryError(RuntimeError):
    """libbnpk.so is missing / not loadable, or no CUDA device: there is no CPU fallback."""


_lib = None


def load_library(path: str = None):
    """dlopen libbnpk.so and attach prototypes.  Does not need a GPU (used by the CPU tests
    that check the exported symbol list)."""
    global _lib
    if _lib is not None and path is None:
        return _lib
    p = path or LIB_PATH
    if not os.path.exists(p):
        raise NativeLibraryError(
            f"{p} not found: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
            "(bionumpy_b200 has no CPU fallback)")
    try:
        lib = ctypes.CDLL(p)
    except OSError as e:  # pragma: no cover
        raise NativeLibraryError(f"cannot load {p}: {e}") from e
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)
        fn.restype = res
        fn.argtypes = args
    if path is None:
        _lib = lib
    return lib


def lib():
    """The library, for compute: additionally requires a CUDA device."""
    if not torch.cuda.is_available():
        raise NativeLibraryError("bionumpy_b200 needs a CUDA device (sm_90a); there is no CPU fallback")
    return load_library()


def check(rc: int):
    if rc == 0:
        return
    msg = load_library().bnpk_last_error().decode()
    if rc in (E_K, E_WINDOW):
        raise AssertionError(msg)  # the reference asserts (kmers.py:69, minimizers.py:50)
    if rc < 0:
        raise ValueError(f"bnpk: {msg} (code {rc})")
    raise RuntimeError(f"bnpk: {msg}")


def stream_ptr():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def ptr(t):
    if t is None:
        return ctypes.c_void_p(0)
    return ctypes.c_void_p(t.data_ptr())


def new_status(device):
    st = torch.empty(ST_WORDS, dtype=torch.int64, device=device)
    check(lib().bnpk_status_init(ptr(st), stream_ptr()))
    return st


_ws_cache = {}


def workspace(n: int, device):
    """Scratch for the look-back kernels: one buffer per (device, stream), grown on demand.  Two streams never
    share look-back state, and a buffer that is replaced is only freed for the stream that used it (the caching
    allocator reuses a block on its own stream in order)."""
    need = int(load_library().bnpk_tile_workspace_bytes(n))
    with torch.cuda.device(device):
        key = (device.type, device.index if device.index is not None else torch.cuda.current_device(),
               torch.cuda.current_stream().cuda_stream)
        ws = _ws_cache.get(key)
        if ws is None or ws.numel() < need:
            ws = torch.empty(max(need, 1 << 16), dtype=torch.uint8, device=device)
            _ws_cache[key] = ws
    return ws
