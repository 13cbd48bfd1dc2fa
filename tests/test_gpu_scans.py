"""The single-pass scans on the GPU against NumPy: ragged row offsets, record format offsets, the per-query run-count
scan of the fused reductions, the interval merge's segmented max and the pileup's coverage and run compaction, each at
item counts around tile borders (2048 items per tile) and over hundreds of tiles."""
import numpy as np
import pytest
import torch

from bionumpy_b200 import _native as nv
from bionumpy_b200 import ops

import pileup_oracle as po
import write_oracle as wo

pytestmark = pytest.mark.gpu

TILE = 2048                      # items per tile of every single-pass scan
INT32_MAX = 2 ** 31 - 1


def _launches(fn):
    lib = nv.load_library()
    torch.cuda.synchronize()
    before = lib.bnpk_launch_count()
    out = fn()
    torch.cuda.synchronize()
    return out, lib.bnpk_launch_count() - before


# --------------------------------------------------------------------------------------------------------------------
# row_offsets
# --------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", [0, 1, TILE - 1, TILE, TILE + 1, 3 * TILE + 5, 200 * TILE + 17])
@pytest.mark.parametrize("shrink", [0, 30, 500])
def test_row_offsets(n, shrink):
    """A quarter of the rows empty and a quarter INT32_MAX long, so that the totals pass 2^32 within a tile and 2^40
    over many tiles."""
    rng = np.random.default_rng(n * 7 + shrink)
    lens = rng.integers(0, 1000, n).astype(np.int64)
    pick = rng.integers(0, 4, n)
    lens[pick == 0] = 0
    lens[pick == 1] = INT32_MAX
    want = np.concatenate([[0], np.cumsum(np.maximum(lens - shrink, 0))])
    got, launches = _launches(lambda: ops.row_offsets(torch.as_tensor(lens.astype(np.int32)).cuda(), shrink))
    assert np.array_equal(got.cpu().numpy(), want)
    assert launches == (1 if n else 0)
    if n > 200 * TILE:
        assert want[TILE] > 2 ** 32 and want[-1] > 2 ** 40


# --------------------------------------------------------------------------------------------------------------------
# format_offsets
# --------------------------------------------------------------------------------------------------------------------
def _field(flat, lens, lut=None):
    lens = np.asarray(lens, dtype=np.int64)
    starts = np.concatenate([[0], np.cumsum(lens)[:-1]])
    return (torch.as_tensor(np.concatenate([flat, np.zeros(16, np.uint8)])).cuda(), torch.as_tensor(starts).cuda(),
            torch.as_tensor(lens.astype(np.int32)).cuda(), lut)


def _entry_starts(text, fmt):
    """The first byte of every entry in the oracle's text: every 4th line of FASTQ, every 2nd line of two-line FASTA,
    and the '>' lines of wrapped FASTA (no sequence line starts with '>')."""
    lines = np.concatenate([[0], np.flatnonzero(text == ord("\n"))[:-1] + 1])
    if fmt == nv.FMT_FASTQ:
        return lines[0::4]
    if fmt == nv.FMT_FASTA:
        return lines[0::2]
    return lines[text[lines] == ord(">")]


@pytest.mark.parametrize("fmt,width", [(nv.FMT_FASTQ, 1), (nv.FMT_FASTA, 1), (nv.FMT_FASTA_WRAPPED, 7)])
@pytest.mark.parametrize("n", [TILE - 1, TILE, TILE + 1, 5 * TILE + 3])
def test_format_offsets(fmt, width, n):
    rng = np.random.default_rng(n + 10 * fmt)
    name_lens, seq_lens = rng.integers(0, 20, n), rng.integers(0, 40, n)
    names = rng.integers(33, 127, int(name_lens.sum())).astype(np.uint8)
    seqs = np.frombuffer(b"ACGT", np.uint8)[rng.integers(0, 4, int(seq_lens.sum()))]
    quals = rng.integers(0, 94, int(seq_lens.sum())).astype(np.uint8)
    if fmt == nv.FMT_FASTQ:
        text = wo.fastq_text(names, name_lens, seqs, seq_lens, quals, seq_lens)
        fields = (_field(names, name_lens), _field(seqs, seq_lens), _field(quals + 33, seq_lens))
    elif fmt == nv.FMT_FASTA:
        text = wo.fasta_text(names, name_lens, seqs, seq_lens)
        fields = (_field(names, name_lens), _field(seqs, seq_lens), None)
    else:
        text = wo.multiline_fasta_text(names, name_lens, seqs, seq_lens, width)
        fields = (_field(names, name_lens), _field(seqs, seq_lens), None)
    starts = _entry_starts(text, fmt)
    assert starts.size == n
    sizes = np.diff(np.concatenate([starts, [text.size]]))
    (offsets, status), launches = _launches(lambda: ops.format_offsets(fmt, width, fields))
    offsets = offsets.cpu().numpy()
    assert np.array_equal(offsets, np.concatenate([[0], np.cumsum(sizes)]))
    assert offsets[-1] == text.size
    assert launches == 2                                    # the status block and the scan
    # a sequence LUT adds the check pass
    lut = torch.as_tensor(np.arange(256, dtype=np.uint8)).cuda()
    fields = (fields[0], fields[1][:3] + (lut,), fields[2])
    (offsets, status), launches = _launches(lambda: ops.format_offsets(fmt, width, fields))
    assert np.array_equal(offsets.cpu().numpy(), np.concatenate([[0], np.cumsum(sizes)]))
    assert int(status[nv.ST_BAD_BASE]) == nv.INT64_MAX
    assert launches == 3


# --------------------------------------------------------------------------------------------------------------------
# runs_reduce: the scan of the run counts per query
# --------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("k", [1, 3, 40])
@pytest.mark.parametrize("delta", [-1, 0, 1])
def test_runs_reduce_count_scan(k, delta):
    """Queries overlapping 0 runs (empty, or outside the track) up to thousands of runs, so that the scanned counts
    vary widely inside and across tiles."""
    n_q = k * TILE + delta
    rng = np.random.default_rng(k * 3 + delta)
    size = 300_000
    dense = po.random_dense(rng, size, np.int64, max_run=3)
    s, e, v = po.runs_of(dense)
    run_starts = torch.as_tensor(np.append(s, size)).cuda()
    values = torch.as_tensor(v.astype(np.int64)).cuda()
    a = rng.integers(-10, size, n_q)
    length = rng.choice([0, 1, 5, 60, 3000, 20000], n_q, p=[0.2, 0.2, 0.2, 0.3, 0.08, 0.02])
    b = a + length
    b[rng.integers(0, n_q, n_q // 50)] = -5                  # stops before starts
    qa, qb = torch.as_tensor(a).cuda(), torch.as_tensor(b).cuda()
    for how, mode in (("max", nv.RUNS_MAX), ("min", nv.RUNS_MIN), ("sum", nv.RUNS_SUM), ("any", nv.RUNS_ANY)):
        got, launches = _launches(lambda: ops.runs_reduce(run_starts, values, qa, qb, mode))
        want = po.reduce_dense(dense, a, b, how)
        assert np.array_equal(got.cpu().numpy(), want.astype(np.int64)), how
        assert launches == 3                                # locate, count scan, reduce


# --------------------------------------------------------------------------------------------------------------------
# interval_merge: the segmented max-scan and the group compaction
# --------------------------------------------------------------------------------------------------------------------
N_MERGE = 300 * TILE + 11


def _merge_rows(rng, same_prev):
    """Starts sorted inside every segment and falling where one starts; stops mostly short, a few long enough to merge
    rows over many tiles.  Segments start at the first and at the last row of tiles, and span 1, 33 and 130 tiles
    (longer than one and than four look-back windows of 32 tiles)."""
    n = N_MERGE
    if same_prev:
        cuts = [0, TILE - 1, TILE, 2 * TILE, 3 * TILE - 1, 36 * TILE - 1, 166 * TILE, 167 * TILE, 167 * TILE + 1,
                168 * TILE - 1]
        cuts += sorted(rng.choice(np.arange(170 * TILE, n), 400, replace=False).tolist())
    else:
        cuts = [0]
    cuts = np.array(cuts + [n])
    seg = np.repeat(np.arange(cuts.size - 1), np.diff(cuts))
    start = np.empty(n, np.int64)
    for i in range(cuts.size - 1):
        m = cuts[i + 1] - cuts[i]
        start[cuts[i]:cuts[i + 1]] = np.sort(rng.integers(0, 30 * m + 1, m))
    stop = start + rng.integers(0, 40, n)
    long_rows = rng.integers(0, n, 60)
    stop[long_rows] += rng.integers(1, 400 * TILE, long_rows.size)
    flags = np.ones(n, np.uint8)
    flags[cuts[:-1]] = 0
    return start, stop, seg, flags


@pytest.mark.parametrize("same_prev", [False, True])
@pytest.mark.parametrize("distance", [0, 5])
def test_interval_merge(same_prev, distance):
    rng = np.random.default_rng(31 + distance + 2 * same_prev)
    start, stop, seg, flags = _merge_rows(rng, same_prev)
    ts, tp = torch.as_tensor(start).cuda(), torch.as_tensor(stop).cuda()
    tf = torch.as_tensor(flags).cuda() if same_prev else None
    (rows, stops, n_out, status), launches = _launches(lambda: ops.interval_merge(ts, tp, tf, distance))
    want_rows, want_stops = po.merge_by_chromosome(seg, start, stop, distance)
    k = int(n_out[0])
    assert k == want_rows.size
    assert np.array_equal(rows[:k].cpu().numpy(), want_rows)
    assert np.array_equal(stops[:k].cpu().numpy(), want_stops)
    assert int(status[nv.ST_BAD_BASE]) == nv.INT64_MAX
    assert launches == 2                                    # the status block and the merge
    # decreasing starts inside a segment: the first one is reported; a decrease where a segment starts is not
    bad = start.copy()
    for r in (250 * TILE + 7, 40 * TILE + TILE - 1, 200 * TILE):
        bad[r] = bad[r - 1] - 1
    if same_prev:
        bad[166 * TILE] = -1                                # a segment's first row
    _, _, _, status = ops.interval_merge(torch.as_tensor(bad).cuda(), tp, tf, distance)
    assert int(status[nv.ST_BAD_BASE]) == 40 * TILE + TILE - 1


def test_interval_merge_launches_without_rows():
    (_, _, n_out, _), launches = _launches(lambda: ops.interval_merge(torch.zeros(0, dtype=torch.int64).cuda(),
                                                                      torch.zeros(0, dtype=torch.int64).cuda()))
    assert int(n_out[0]) == 0
    assert launches == 1                                    # the status block only


# --------------------------------------------------------------------------------------------------------------------
# pileup_runs: coverage and run compaction
# --------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("k", [1, 200])
@pytest.mark.parametrize("delta", [-2, 0, 2])
@pytest.mark.parametrize("mode", [nv.PILEUP_COUNT, nv.PILEUP_ANY])
def test_pileup_runs(k, delta, mode):
    """2048k - 2, 2048k and 2048k + 2 event keys (two per interval), on few positions, so that groups of equal keys
    straddle thread and tile borders."""
    n = (k * TILE + delta) // 2
    rng = np.random.default_rng(k * 5 + delta + mode)
    size = 40 * k + 10
    a = rng.integers(0, 40 * k, n)
    b = np.minimum(a + rng.integers(0, 5, n), size)
    keys = np.sort(np.concatenate([a << 1 | 1, b << 1]))
    assert keys.size == k * TILE + delta
    (starts, values, n_runs), launches = _launches(lambda: ops.pileup_runs(torch.as_tensor(keys).cuda(), size, mode))
    s, e, v = po.event_runs(a, b, size, mode == nv.PILEUP_ANY)
    r = int(n_runs[0])
    assert r == s.size
    assert np.array_equal(starts[:r + 1].cpu().numpy(), np.append(s, size))
    assert np.array_equal(values[:r].cpu().numpy(), v.astype(np.int64))
    assert launches == 1
