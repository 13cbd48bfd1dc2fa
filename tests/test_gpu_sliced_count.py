"""The fused count fed in slices (bnpk_chunk_kmer_count with consecutive [slice_begin, slice_end) ranges of one resident
buffer, one workspace and one status block), and the host pipeline built on that contract, on every kernel route.

A sliced count must give what one launch over the whole chunk gives, bit for bit: the histogram and all status words.
The slice driver can poison the device buffer first and copy each slice's bytes in only just before its call, as the
pipeline does while the next slice is still in flight, so any read past `slice_end` changes the result.  The one-shot
launch of every (input, route) is itself checked against the oracle."""
import numpy as np
import pytest
import torch
from collections import namedtuple

from oracle import bnp_oracle as o

gpu = pytest.mark.gpu

TILE, MiB = 16384, 1 << 20
HIST_AUTO, HIST_GLOBAL = 0, 2
ENC_ACGT, ENC_ACTG, ENC_LUT = 0, 1, 3

# Each case and the kernel its call must reach (the *_eligible tests of tile_ws_kernel.cu / tile_tma_kernel.cu and
# launch_count in tile_kernels.cu).  Kernel names as the profiler reports them, template arguments normalised.
Route = namedtuple("Route", "k bins window hist_mode shift kernels")
TILE_SMEM_K, TILE_SMEM_MZ, TILE_GLOBAL_MZ = ("bnpk::tile_kernel<1, 0, true, false>", "bnpk::tile_kernel<1, 0, true, true>",
                                             "bnpk::tile_kernel<1, 0, false, true>")
ROUTES = {
    "ws_exact": Route(5, 1024, 0, HIST_AUTO, 0, ("bnpk::ws::tile_ws_kernel<0>",)),
    "ws": Route(31, 1 << 14, 0, HIST_AUTO, 0, ("bnpk::ws::tile_ws_kernel<0>",)),
    "wsm": Route(31, 1 << 14, 41, HIST_AUTO, 0, ("bnpk::wsm::tile_ws_kernel<0>",)),           # 11 k-mers per window
    "wsm_widest": Route(7, 100, 18, HIST_AUTO, 0, ("bnpk::wsm::tile_ws_kernel<0>",)),         # 12 k-mers per window
    "tma": Route(21, 1 << 20, 0, HIST_AUTO, 0, ("bnpk::tma::tile_tma_kernel<0, 0>",)),
    "tma_modulo": Route(31, 1000003, 0, HIST_AUTO, 0, ("bnpk::tma::tile_tma_kernel<0, 0>",)),
    "tma_global": Route(31, 1 << 14, 0, HIST_GLOBAL, 0, ("bnpk::tma::tile_tma_kernel<0, 0>",)),
    "scratch": Route(31, 1 << 24, 0, HIST_AUTO, 0, ("bnpk::tma::tile_tma_kernel<0, 2>", "bnpk::widen_add_kernel")),
    "scratch_modulo": Route(31, 5000011, 0, HIST_AUTO, 0, ("bnpk::tma::tile_tma_kernel<0, 2>", "bnpk::widen_add_kernel")),
    "tile_smem": Route(31, 1 << 15, 0, HIST_AUTO, 0, (TILE_SMEM_K,)),
    "tile_w13": Route(31, 1 << 14, 43, HIST_AUTO, 0, (TILE_SMEM_MZ,)),                       # 13 k-mers per window
    "tile_global_minz": Route(31, 1 << 20, 41, HIST_AUTO, 0, (TILE_GLOBAL_MZ,)),
    "unaligned": Route(31, 1 << 14, 0, HIST_AUTO, 3, (TILE_SMEM_K,)),
    "unaligned_minz": Route(15, 1 << 12, 25, HIST_AUTO, 5, (TILE_SMEM_MZ,)),
}
ALIGNED = [name for name, r in ROUTES.items() if r.shift == 0]
# exact 7-mers take the warp-specialised kernel in every encoding (ACTG mode, LUT mode)
ALL_ROUTES = dict(ROUTES, ws_actg=Route(7, 4 ** 7, 0, HIST_AUTO, 0, ("bnpk::ws::tile_ws_kernel<",)))
COUNT_KERNELS = ("bnpk::ws::", "bnpk::wsm::", "bnpk::tma::", "bnpk::tile_kernel<1,", "bnpk::widen_add_kernel")

SCHEDULES = ["one_shot", "step16384", "step18432", "step18431", "step100003", "step1MiB", "step4MiB", "first7",
             "random", "empty_final"]


def schedule(name, n):
    """The calls of a slicing schedule: (slice_begin, slice_end, final_slice).  The last call is always final."""
    def steps(first, step):
        cuts = [0] + ([first] if first else [])
        while cuts[-1] < n:
            cuts.append(min(n, cuts[-1] + step))
        return cuts
    if name == "one_shot":
        cuts = [0, n]
    elif name.startswith("step"):
        cuts = steps(0, {"1MiB": MiB, "4MiB": 4 * MiB}.get(name[4:]) or int(name[4:]))
    elif name == "first7":                                   # the first slice ends inside the first header line
        cuts = steps(7, MiB)
    elif name == "random":                                   # repeated cuts make empty slices, [0, 0) among them
        rng = np.random.default_rng(n)
        c = rng.integers(0, n + 1, 25)
        cuts = [0, 0] + sorted(int(x) for x in np.concatenate([c, c[:5]])) + [n]
    elif name == "empty_final":                              # every byte in non-final calls, then [n, n) final
        cuts = steps(0, MiB)
        return [(b, e, False) for b, e in zip(cuts, cuts[1:])] + [(n, n, True)]
    else:
        raise ValueError(name)
    return [(b, e, i == len(cuts) - 2) for i, (b, e) in enumerate(zip(cuts, cuts[1:]))]


# ---- inputs -------------------------------------------------------------------------------------------------------------
def fastq_bytes(rng, lens, lower_frac=0.0, eol=b"\n", first_eol=None):
    """FASTQ records with the given read lengths (quality lines start with '@' and '+' now and then)."""
    total = int(lens.sum())
    seq = rng.choice(np.frombuffer(b"ACGT", dtype=np.uint8), size=total)
    if lower_frac:
        seq = np.where(rng.random(total) < lower_frac, seq + 32, seq).astype(np.uint8)
    qual = rng.integers(33, 74, size=total, dtype=np.uint8)
    parts, off = [], 0
    for r, L in enumerate(lens.tolist()):
        e = first_eol if (r == 0 and first_eol is not None) else eol
        parts += [b"@read%d x" % r, e, seq[off:off + L].tobytes(), e, b"+", e, qual[off:off + L].tobytes(), e]
        off += L
    return np.frombuffer(b"".join(parts), dtype=np.uint8).copy()


def fasta_bytes(rng, lens):
    seq = rng.choice(np.frombuffer(b"ACGTacgt", dtype=np.uint8), size=int(lens.sum()))
    parts, off = [], 0
    for r, L in enumerate(lens.tolist()):
        parts += [b">contig%d x\n" % r, seq[off:off + L].tobytes(), b"\n"]
        off += L
    return np.frombuffer(b"".join(parts), dtype=np.uint8).copy()


Input = namedtuple("Input", "data lpe header check_plus error")      # error: None or (kind, expected status value)


def _ragged(seed, n_records):
    rng = np.random.default_rng(seed)
    lens = rng.integers(0, 401, n_records)
    lens[-1] = 300                                            # a last read long enough to truncate inside
    return fastq_bytes(rng, lens, lower_frac=0.1)


def _with_error(kind):
    """A ragged chunk with one error in its last third: a bad base in a row that a tile boundary (so a cut of every
    16384-byte schedule) crosses, a bad header or a bad '+' line."""
    chunk = _ragged(71, 5000)
    _, starts, lens = o.fastq_split(chunk)
    n = chunk.size
    if kind == "base":
        s, e = starts[:, 1], starts[:, 1] + lens[:, 1]
        cut = (s // TILE + 1) * TILE
        r = int(np.flatnonzero((s > 2 * n // 3) & (cut < e - 1))[0])
        pos = int(cut[r] - s[r])
        chunk[s[r] + pos] = ord("N")
        with pytest.raises(o.OracleEncodingError) as ex:
            o.encode_flat(o.gather_rows(chunk, starts[:, 1], lens[:, 1]), o.alphabet_lut())
        assert ex.value.offset == int(lens[:r, 1].sum()) + pos
        return Input(chunk, 4, "@", True, ("base", (r, pos)))
    entry = int(np.searchsorted(starts[:, 0], (3 if kind == "header" else 4) * n // 5))
    if kind == "header":
        chunk[starts[entry, 0] - 1] = ord("#")
    else:
        chunk[starts[entry, 2]] = ord("-")
    with pytest.raises(o.OracleFormatException) as ex:
        o.fastq_split(chunk)
    assert ex.value.line_number // 4 == entry
    return Input(chunk, 4, "@", True, (kind, entry))


def _build_input(name):
    fq = lambda data: Input(data, 4, "@", True, None)
    if name == "ragged":                                      # F1, ~4 MB
        return fq(_ragged(61, 9500))
    if name == "synthetic":                                   # F1, ~12.7 MB: several tiles per CTA in every slice
        return fq(o.synthetic_fastq(0, 40000))
    if name in ("crlf", "crlf_mixed"):                        # F2: CRLF; or the first record LF, all later ones CRLF
        rng = np.random.default_rng(62)
        return fq(fastq_bytes(rng, rng.integers(0, 301, 5000), eol=b"\r\n", first_eol=b"\n" if name == "crlf_mixed" else None))
    if name == "long":                                        # F3: deferred rows that cross slice cuts
        rng = np.random.default_rng(63)
        lens = rng.integers(2500, 60001, 24)
        lens[11] = 150_000
        return fq(fastq_bytes(rng, lens))
    if name.startswith("trunc_"):                             # F4
        chunk = _ragged(64, 6000)
        _, starts, _ = o.fastq_split(chunk)
        end = {"trunc_seq": starts[-1, 1] + 150, "trunc_qual": starts[-1, 3] + 150, "trunc_nl": chunk.size - 1}[name]
        return fq(chunk[:end].copy())
    if name == "fasta":                                       # F5: two-line FASTA, a few rows of 3-20 kb
        rng = np.random.default_rng(65)
        lens = rng.integers(0, 900, 3000)
        lens[::40] = rng.integers(3000, 20001, lens[::40].size)
        return Input(fasta_bytes(rng, lens), 2, ">", False, None)
    if name.startswith("bad_"):                               # F6
        return _with_error(name[4:])
    raise ValueError(name)


FAMILIES = ["crlf", "crlf_mixed", "long", "trunc_seq", "trunc_qual", "trunc_nl", "fasta", "bad_base", "bad_header",
            "bad_plus"]
FAMILY_ROUTES = ["ws", "wsm", "tma", "scratch", "tile_smem", "unaligned"]
FAMILY_SCHEDULES = ["step16384", "first7", "random"]

_inputs, _device_inputs, _oracles, _refs, _poisons = {}, {}, {}, {}, {}


def get_input(name):
    if name not in _inputs:
        _inputs[name] = _build_input(name)
    return _inputs[name]


def device_input(name):
    if name not in _device_inputs:
        _device_inputs[name] = torch.from_numpy(get_input(name).data).cuda()
    return _device_inputs[name]


def oracle(name, k, bins, window, alphabet="ACGT"):
    """(hist, n_records, n_complete_bytes, n_bases) of the reference path, once per (input, k, bins, window)."""
    key = (name, k, bins, window, alphabet)
    if key not in _oracles:
        inp = get_input(name)
        size, starts, lens = (o.fastq_split if inp.lpe == 4 else o.two_line_fasta_split)(inp.data)
        lut = o.alphabet_lut(alphabet)
        codes = o.encode_flat(o.gather_rows(inp.data, starts[:, 1], lens[:, 1]), lut)
        vals, _ = o.get_minimizers_fast(codes, lens[:, 1], k, window) if window else o.get_kmers(codes, lens[:, 1], k)
        hist = o.count_encoded_flat(vals, bins) if bins == 4 ** k else o.count_bucketed_flat(vals, bins)
        _oracles[key] = (torch.from_numpy(hist).cuda(), starts.shape[0], size, int(lens[:, 1].sum()))
    return _oracles[key]


def poison(kind, size):
    """Device bytes that change the result if a kernel reads them: all '\n' (line counts, the line phase) or a
    different valid FASTQ (k-mers)."""
    key = (kind, size)
    if key not in _poisons:
        if kind == "newlines":
            _poisons[key] = torch.full((size,), 10, dtype=torch.uint8, device="cuda")
        else:
            from bionumpy_b200 import ops
            _poisons[key] = ops.synth_fastq(size // 317 + 1, first_record=7_000_000)[:size].clone()
    return _poisons[key]


def count_sliced(src, calls, route, inp, enc=ENC_ACGT, lut=None, poison_kind=None, hist0=None):
    """Feed the device chunk `src` to bnpk_chunk_kmer_count as `calls`, on one status block and one workspace.
    The chunk sits `route.shift` bytes into its buffer.  With `poison_kind`, the buffer starts out poisoned and each
    slice's bytes are copied in (on the same stream) just before its call.  `hist0` pre-fills the histogram."""
    from bionumpy_b200 import _native as nv
    n = src.numel()
    size = n + route.shift + 64
    if poison_kind is None:
        buf = torch.zeros(size, dtype=torch.uint8, device="cuda")
    else:
        buf = poison(poison_kind, size).clone()
    chunk = buf[route.shift: route.shift + n]
    if poison_kind is None:
        chunk.copy_(src)
    hist = hist0.clone() if hist0 is not None else torch.zeros(route.bins, dtype=torch.int64, device="cuda")
    status = nv.new_status(src.device)
    ws = nv.workspace(n, src.device)
    for b, e, final in calls:
        if poison_kind is not None and e > b:
            chunk[b:e].copy_(src[b:e])
        nv.check(nv.lib().bnpk_chunk_kmer_count(
            nv.ptr(chunk), n, b, e, int(final), inp.lpe, ord(inp.header), int(inp.check_plus), -1, enc, nv.ptr(lut),
            route.k, route.window, route.bins, route.hist_mode, nv.ptr(hist), nv.ptr(status), nv.ptr(ws), ws.numel(),
            nv.stream_ptr()))
    return hist, status.cpu().tolist()


def prefill(bins, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.randint(0, 1 << 40, (bins,), generator=g, device="cuda", dtype=torch.int64)


def check_status(st, inp, n_records=None, size=None, n_bases=None, n_values=None):
    """The one-shot status against the oracle: counts, and errors exactly where the oracle raises."""
    from bionumpy_b200 import ops
    s = ops.ScanStatus(st)
    if n_records is not None:
        assert (s.n_records, s.n_complete_bytes, s.n_bases, s.n_values) == (n_records, size, n_bases, n_values)
    kind, want = inp.error or (None, None)
    assert s.bad_base() == (want if kind == "base" else None)
    assert s.bad_header_entry == (want if kind == "header" else None)
    assert s.bad_plus_entry == (want if kind == "plus" else None)
    assert not s.overflow


def reference(name, route_name, enc=ENC_ACGT):
    """One launch over the whole chunk on the route, checked against the oracle (input F6: its errors only)."""
    key = (name, route_name, enc)
    if key not in _refs:
        inp, route = get_input(name), ALL_ROUTES[route_name]
        lut = torch.from_numpy(o.alphabet_lut("ACTG")).cuda() if enc == ENC_LUT else None
        src = device_input(name)
        hist, st = count_sliced(src, schedule("one_shot", src.numel()), route, inp, enc, lut)
        if inp.error is None:
            want, n_records, size, n_bases = oracle(name, route.k, route.bins, route.window,
                                                    "ACGT" if enc == ENC_ACGT else "ACTG")
            assert torch.equal(hist, want), (name, route_name)
            check_status(st, inp, n_records, size, n_bases, int(want.sum()))
        else:
            check_status(st, inp)
        _refs[key] = (hist, st)
    return _refs[key]


def diff_words(st, ref):
    from bionumpy_b200 import _native as nv
    names = {getattr(nv, a): a for a in dir(nv) if a.startswith("ST_") and a != "ST_WORDS"}
    return [(names.get(i, i), a, b) for i, (a, b) in enumerate(zip(st, ref)) if a != b]


def check_sliced(name, route_name, sched, poisons, enc=ENC_ACGT):
    inp, route = get_input(name), ALL_ROUTES[route_name]
    ref_hist, ref_st = reference(name, route_name, enc)
    lut = torch.from_numpy(o.alphabet_lut("ACTG")).cuda() if enc == ENC_LUT else None
    src = device_input(name)
    calls = schedule(sched, src.numel())
    hist0 = prefill(route.bins)
    for p in poisons:
        hist, st = count_sliced(src, calls, route, inp, enc, lut, poison_kind=p, hist0=hist0)
        assert torch.equal(hist, hist0 + ref_hist), (name, route_name, sched, p)
        assert st == ref_st, (name, route_name, sched, p, diff_words(st, ref_st))


# ---- sliced launches ----------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("sched", SCHEDULES)
@pytest.mark.parametrize("route", list(ROUTES))
@pytest.mark.parametrize("name", ["ragged", "synthetic"])
def test_sliced_matches_one_shot(name, route, sched):
    """F1 on every route and schedule: with the whole buffer resident, and with the bytes past each slice poisoned."""
    check_sliced(name, route, sched, [None, "newlines", "fastq"])


@gpu
@pytest.mark.parametrize("sched", FAMILY_SCHEDULES)
@pytest.mark.parametrize("route", FAMILY_ROUTES)
@pytest.mark.parametrize("name", FAMILIES)
def test_families_sliced(name, route, sched):
    """CRLF, long deferred rows, truncated last records, two-line FASTA and late errors, cut by slices, poisoned."""
    check_sliced(name, route, sched, ["newlines", "fastq"])


@gpu
@pytest.mark.parametrize("sched", FAMILY_SCHEDULES)
@pytest.mark.parametrize("enc", [ENC_ACTG, ENC_LUT])
@pytest.mark.parametrize("route", ["ws_actg", "tma"])
def test_encodings_sliced(route, enc, sched):
    """ACTG mode and LUT mode (an ACTG table), on the warp-specialised and the bulk-copy kernel."""
    check_sliced("ragged", route, sched, ["fastq"], enc)


def test_slice_schedules_cover_the_chunk():
    """Every schedule feeds consecutive slices that cover [0, n) and ends with exactly one final call."""
    for n in (7, 18431, 4_000_003, 12_680_000):
        for sched in SCHEDULES:
            calls = schedule(sched, n)
            assert calls[0][0] == 0 and calls[-1][1] == n and calls[-1][2]
            assert sum(c[2] for c in calls) == 1
            assert all(b <= e for b, e, _ in calls) and all(a[1] == b[0] for a, b in zip(calls, calls[1:]))
    assert any(b == e for b, e, _ in schedule("random", 4_000_003))
    assert schedule("empty_final", 4_000_003)[-1] == (4_000_003, 4_000_003, True)
    assert schedule("first7", 4_000_003)[0] == (0, 7, False)


# ---- which kernel each case reaches -------------------------------------------------------------------------------------
def _normalise(name):
    return name.replace("(int)", "").replace("(bool)1", "true").replace("(bool)0", "false")


PROFILE_ATTEMPTS = 5


@gpu
def test_each_case_reaches_its_kernel():
    """Pins the route table: a change to the eligibility tests must not silently move a case to another kernel.

    Late in a long test process the CUDA profiler can lose the records of a session's first kernels (the fills, the
    status init and the count kernel) while it keeps the later ones of the same call (the deferred-row and finalize
    kernels).  A call's route is fixed by the call alone, so a session that lacks a kernel of the route is repeated, up
    to PROFILE_ATTEMPTS sessions per case.  Every session must show no count kernel outside the route, and one of them
    must show every kernel of the route."""
    from torch.profiler import profile, ProfilerActivity
    inp = get_input("ragged")
    src = device_input("ragged")
    any_kernel = False
    for route_name, route in ROUTES.items():
        want = {c for c in COUNT_KERNELS if any(c in kern for kern in route.kernels)}
        sessions = []
        for _ in range(PROFILE_ATTEMPTS):
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                count_sliced(src, schedule("one_shot", src.numel()), route, inp)
                torch.cuda.synchronize()
            names = {_normalise(e.key) for e in prof.key_averages()}
            any_kernel |= any("bnpk::" in n for n in names)
            launched = {c for c in COUNT_KERNELS if any(c in n for n in names)}
            assert launched <= want, (route_name, sorted(names))
            sessions.append(sorted(names))
            if all(any(kern in n for n in names) for kern in route.kernels):
                break
        else:
            if not any_kernel:
                pytest.skip("the profiler recorded no CUDA kernels")
            raise AssertionError((route_name, route.kernels, sessions))


# ---- the host pipeline --------------------------------------------------------------------------------------------------
def _host(name):
    return torch.from_numpy(get_input(name).data).pin_memory()


def _pipe_count(pipe, name, route_name, hist0=None, enc=ENC_ACGT, lut_host=None):
    inp, route = get_input(name), ALL_ROUTES[route_name]
    hist = hist0.clone() if hist0 is not None else torch.zeros(route.bins, dtype=torch.int64, device="cuda")
    st = pipe.kmer_count(_host(name), route.k, hist, window_size=route.window, lines_per_entry=inp.lpe,
                         header_char=ord(inp.header), check_plus=inp.check_plus, enc_mode=enc, lut_host=lut_host,
                         hist_mode=route.hist_mode)
    return hist, st.words


@gpu
@pytest.mark.parametrize("slice_bytes", [1, MiB])
@pytest.mark.parametrize("route", ALIGNED)
def test_pipeline_matches_one_shot(route, slice_bytes):
    """Every aligned route through the pipeline (slices of one tile, or 1 MiB), into a pre-filled histogram."""
    from bionumpy_b200 import ops
    ref_hist, ref_st = reference("ragged", route)
    pipe = ops.HostPipeline(get_input("ragged").data.size, slice_bytes=slice_bytes)
    hist0 = prefill(ALL_ROUTES[route].bins, 1)
    hist, st = _pipe_count(pipe, "ragged", route, hist0)
    pipe.close()
    assert torch.equal(hist, hist0 + ref_hist)
    assert st == ref_st, diff_words(st, ref_st)


@gpu
@pytest.mark.parametrize("slice_bytes", [1, MiB])
@pytest.mark.parametrize("enc", [ENC_ACTG, ENC_LUT])
def test_pipeline_encodings(enc, slice_bytes):
    """ACTG mode, and LUT mode through `lut_host` (the pipeline uploads the table)."""
    from bionumpy_b200 import ops
    lut_host = torch.from_numpy(o.alphabet_lut("ACTG")) if enc == ENC_LUT else None
    pipe = ops.HostPipeline(get_input("ragged").data.size, slice_bytes=slice_bytes)
    for route in ("ws_actg", "tma"):
        ref_hist, ref_st = reference("ragged", route, enc)
        hist, st = _pipe_count(pipe, "ragged", route, enc=enc, lut_host=lut_host)
        assert torch.equal(hist, ref_hist), route
        assert st == ref_st, (route, diff_words(st, ref_st))
    pipe.close()


@gpu
@pytest.mark.parametrize("name", ["crlf", "crlf_mixed"])
def test_pipeline_crlf(name):
    from bionumpy_b200 import ops
    pipe = ops.HostPipeline(get_input(name).data.size, slice_bytes=1)
    for route in ("ws", "tma", "scratch"):
        ref_hist, ref_st = reference(name, route)
        hist, st = _pipe_count(pipe, name, route)
        assert torch.equal(hist, ref_hist), route
        assert st == ref_st and ops.ScanStatus(st).cr, (route, diff_words(st, ref_st))
    pipe.close()


@gpu
def test_pipeline_reused_across_chunks():
    """One pipeline object for chunks of different sizes, errors, tables and encodings, then an empty chunk."""
    from bionumpy_b200 import ops
    pipe = ops.HostPipeline(get_input("synthetic").data.size, slice_bytes=MiB)

    def same(name, route, enc=ENC_ACGT, lut_host=None):
        ref_hist, ref_st = reference(name, route, enc)
        hist, st = _pipe_count(pipe, name, route, enc=enc, lut_host=lut_host)
        assert torch.equal(hist, ref_hist), (name, route)
        assert st == ref_st, (name, route, diff_words(st, ref_st))

    same("synthetic", "ws")
    same("trunc_qual", "ws")             # a smaller, different chunk: the bigger one's bytes lie past n
    same("bad_base", "ws")
    same("ragged", "ws")                 # clean status after an error
    same("ragged", "scratch")
    same("ragged", "scratch_modulo")
    same("ragged", "tma", ENC_LUT, torch.from_numpy(o.alphabet_lut("ACTG")))
    same("ragged", "tma")
    hist = prefill(1 << 14, 2)
    want = hist.clone()
    empty = torch.empty(0, dtype=torch.uint8)
    _, empty_status = ops.chunk_kmer_count(torch.empty(0, dtype=torch.uint8, device="cuda"), 31, 1 << 14, hist=want)
    for chunk in (empty, _host("ragged")[:0]):
        st = pipe.kmer_count(chunk, 31, hist)
        assert st.words == empty_status.cpu().tolist()
        assert torch.equal(hist, want)
    pipe.close()


@gpu
def test_pipeline_rejects_chunk_over_capacity():
    from bionumpy_b200 import ops
    pipe = ops.HostPipeline(1 << 16, slice_bytes=1)
    hist = torch.zeros(1 << 14, dtype=torch.int64, device="cuda")
    with pytest.raises(ValueError):
        pipe.kmer_count(torch.from_numpy(o.synthetic_fastq(0, 300)), 31, hist)
    pipe.close()


# ---- argument checks (no GPU) -------------------------------------------------------------------------------------------
def test_chunk_count_rejects_bad_arguments_before_touching_memory():
    """Documented error codes, with null pointers everywhere: nothing is read or launched before the checks."""
    from bionumpy_b200 import _native as nv
    lib = nv.load_library()
    n = 100000
    ws_bytes = int(lib.bnpk_tile_workspace_bytes(n))

    def call(n=n, b=0, e=n, lpe=4, k=31, window=0, ws=ws_bytes, enc=ENC_ACGT):
        return lib.bnpk_chunk_kmer_count(None, n, b, e, 1, lpe, ord("@"), 1, -1, enc, None, k, window, 1 << 14,
                                         HIST_AUTO, None, None, None, ws, None)

    assert call(e=n + 1) == nv.E_BADARG                       # slice_end > n
    assert call(b=50, e=49) == nv.E_BADARG                    # slice_begin > slice_end
    assert call(lpe=3) == nv.E_BADARG
    assert call(ws=ws_bytes - 1) == nv.E_WORKSPACE
    assert call(k=21, window=20) == nv.E_WINDOW
    assert call(k=32) == nv.E_K
    assert call(enc=-1) == call(enc=4) == nv.E_BADARG
    assert call(enc=nv.ENC_LUT) == nv.E_BADARG                # without lut256
    assert call(n=0, e=0, ws=int(lib.bnpk_tile_workspace_bytes(0))) == 0     # an empty chunk does nothing
