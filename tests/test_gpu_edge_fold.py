"""Edge windows of the folded path (one tagset, regular shard, no strict order).

A segment's first and last window may continue in the neighbouring segments of its series.  A folding lane group whose
lanes share one time grid adds those windows to its shared-memory bucket accumulators like its interior windows; segments
that cannot (lanes on different grids, a segment inside one window, segments the fused kernel leaves over) keep the
ordered edge stitch.  Both kinds meet in one bucket, so every case runs run_both: strict order and the oracle bitwise,
then the folded order (sums within SUM_RTOL, everything else bitwise)."""
import numpy as np
import pytest

from opengemini_b200 import AggQuery, Shard
from opengemini_b200 import _lib as L
import oracle
from test_gpu_parity import run_both

pytestmark = pytest.mark.gpu

T0 = 1_700_000_000_000_000_000
SEC = 1_000_000_000
ALL6 = ["count", "sum", "min", "max", "first", "last"]


@pytest.fixture(scope="module", autouse=True)
def _device():
    Shard.init(0)


def _open(series):
    """series: list of series, each a list of (times int64[], values float64[]) segments in time order."""
    pages, tpages, tmins, tmaxs, ssb = [], [], [], [], [0]
    for segs in series:
        for t, v in segs:
            pages.append(oracle.field_page_encode(L.TYPE_FLOAT, np.asarray(v, np.float64)))
            tpages.append(oracle.time_page_encode(t)); tmins.append(int(t[0])); tmaxs.append(int(t[-1]))
        ssb.append(ssb[-1] + len(segs))
    blob, offs, lens, pos = [], [], [], 0
    for p in pages + tpages:
        offs.append(pos); lens.append(p.size); blob.append(p); pos += p.size
    nseg = ssb[-1]
    sh = Shard.open(np.concatenate(blob), np.arange(1, len(series) + 1), ssb, tmins, tmaxs,
                    [("v", L.TYPE_FLOAT, offs[:nseg], lens[:nseg])], offs[nseg:], lens[nseg:])
    return sh, oracle.shard_desc_from_export(sh.export())


def _grid(n_series, n_seg, rows, values, start=lambda s: 0, dt=lambda s: SEC, jitter=lambda s, g: False):
    """n_seg segments of `rows` rows per series; series s starts at T0 + start(s) with cadence dt(s).  values(s, t) gives the
    values at times t; jitter(s, g) gives segment g irregular times (a Simple8b time page: not taken by the fused kernel)."""
    out = []
    for s in range(n_series):
        segs = []
        for g in range(n_seg):
            t = T0 + start(s) + (np.arange(rows, dtype=np.int64) + g * rows) * dt(s)
            if jitter(s, g):
                t = t + (np.arange(rows, dtype=np.int64) % 3) * 1000
            segs.append((t, values(s, t)))
        out.append(segs)
    return out


def _rng_values(seed, bits=20):
    rng = np.random.default_rng(seed)
    return lambda s, t: 100.0 + np.floor(rng.random(t.size) * 2.0**bits) / 2.0**bits


def _stats(sh, calls, iv, tmin, tmax):
    q = AggQuery(sh, calls, iv, tmin, tmax).run()
    st = q.stats()
    q.close()
    return st


def test_common_case_stays_folded():
    """Aligned series, 1000-row segments, 60 s windows: every segment's head and tail are folded in the warp."""
    series = _grid(70, 4, 1000, _rng_values(1))
    sh, sd = _open(series)
    tmax = T0 + 3999 * SEC
    for calls in ([("sum", 0), ("count", 0), ("max", 0)], [("min", 0)], [(f, 0) for f in ALL6]):
        run_both(sh, sd, calls, 60 * SEC, T0, tmax, f"aligned {calls}")
    st = _stats(sh, [("sum", 0), ("count", 0), ("max", 0)], 60 * SEC, T0, tmax)
    assert st["path"] == 3 and st["per_series_cells_used"] == 0, st
    sh.close()


@pytest.mark.parametrize("rows", [20, 7])
def test_windows_that_span_three_or_more_segments(rows):
    """Segments shorter than a window: some segments lie inside one window and keep the ordered edge stitch, their
    neighbours fold their edges in the warp."""
    series = _grid(40, 30, rows, _rng_values(2))
    sh, sd = _open(series)
    tmax = T0 + (30 * rows - 1) * SEC
    for iv in (60 * SEC, 45 * SEC, 2 * rows * SEC):
        for calls in ([("sum", 0), ("count", 0), ("max", 0)], [(f, 0) for f in ALL6]):
            run_both(sh, sd, calls, iv, T0, tmax, f"short segments rows={rows} iv={iv} {calls}")
    run_both(sh, sd, [("min", 0), ("sum", 0)], 60 * SEC, T0 + 33 * SEC + 1, T0 + (20 * rows) * SEC - 1, "short segments cut")
    sh.close()


def test_leftover_segments_meet_folded_edges():
    """Some segments are not taken by the fused kernel (irregular times -> Simple8b time page; constant values -> a 'same'
    page): their edge windows go through the ordered stitch while their neighbours' edges are folded in the warp, and both
    land in the same buckets."""
    vals = _rng_values(3)

    def values(s, t):
        v = vals(s, t)
        return np.full(t.size, 100.25) if (s % 5 == 1 and (t[0] - T0) // SEC // 1000 == 2) else v

    series = _grid(66, 5, 1000, values, jitter=lambda s, g: s % 7 == 3 and g in (1, 3))
    sh, sd = _open(series)
    tmax = T0 + 4999 * SEC
    st = _stats(sh, [("sum", 0)], 60 * SEC, T0, tmax)
    assert st["path"] == 3 and st["general_segments"] > 0, st
    for calls in ([("sum", 0), ("count", 0), ("max", 0)], [(f, 0) for f in ALL6], [("first", 0)], [("last", 0)]):
        run_both(sh, sd, calls, 60 * SEC, T0, tmax, f"leftovers {calls}")
    run_both(sh, sd, [("max", 0), ("count", 0)], 45 * SEC, T0 + 999 * SEC, T0 + 3001 * SEC, "leftovers cut")
    sh.close()


def test_lanes_on_different_grids_in_one_group():
    """Every segment index covers the same time range in every series, but cadences differ (1 s, 3 s, 9 s over 999 s).
    Lane groups are cut from the streams sorted by length, and with 34/33/33 series per cadence two groups of every segment
    index mix cadences: they cannot fold (their lanes reach windows at different rows) and keep the edge stitch and the
    per-series cells, while the groups of one cadence fold."""
    cad = [1, 3, 9]
    rows_of = {1: 1000, 3: 334, 9: 112}
    vals = _rng_values(4)
    series = []
    for s in range(100):
        c = cad[s % 3]
        segs = []
        for g in range(4):
            t = T0 + g * 1000 * SEC + np.arange(rows_of[c], dtype=np.int64) * c * SEC
            segs.append((t, vals(s, t)))
        series.append(segs)
    sh, sd = _open(series)
    tmax = T0 + 3999 * SEC
    st = _stats(sh, [("sum", 0), ("count", 0)], 60 * SEC, T0, tmax)
    assert st["path"] == 3 and st["per_series_cells_used"] == 1, st  # folded plan, and some lane groups mix cadences
    for calls in ([("sum", 0), ("count", 0), ("max", 0)], [(f, 0) for f in ALL6]):
        run_both(sh, sd, calls, 60 * SEC, T0, tmax, f"cadences {calls}")
        run_both(sh, sd, calls, 60 * SEC, T0 + 500 * SEC + 1, T0 + 3300 * SEC, f"cadences cut {calls}")
    sh.close()


@pytest.mark.parametrize("before_x", [5, 1, 50])
def test_head_runs_of_neighbouring_segment_indices_in_one_bucket(before_x):
    """Two segment indices lead runs in one bucket of one block of 32 series.  Windows (60 s) are aligned to the epoch; X is
    the window that holds the last 30 s of segment 0 and the first 30 s of segment 1, and the range starts `before_x`
    seconds before X, in the second-to-last bucket of segment 0.  Series s % 3 == 0 have a 9 s cadence: for before_x = 5
    and 1 their first row in range is in X, so their segment 0 lies inside one bucket and leads a run at X from segment
    index 0.  The other series have a 1 s cadence: their segment 0 spans X-1 and X and folds its edges in the warp, and for
    s % 3 == 1 segment 1 is a constant page that the fused kernel leaves over, so head(1) leads a run at X from segment
    index 1 in the same block."""
    iv = 60 * SEC
    x_start = T0 + (-T0) % iv + 16 * iv      # a window boundary about 1000 s after T0
    s0 = x_start - 970 * SEC                 # segment g covers [s0 + 1000 g s, s0 + 1000 g s + 999 s]
    vals = _rng_values(9)
    series = []
    for s in range(96):
        c, n = (9, 112) if s % 3 == 0 else (1, 1000)
        segs = []
        for g in range(3):
            t = s0 + g * 1000 * SEC + np.arange(n, dtype=np.int64) * c * SEC
            v = np.full(n, 100.5) if (s % 3 == 1 and g == 1) else vals(s, t)
            segs.append((t, v))
        series.append(segs)
    sh, sd = _open(series)
    tmin, tmax = x_start - before_x * SEC, s0 + 2999 * SEC
    st = _stats(sh, [("sum", 0)], iv, tmin, tmax)
    assert st["path"] == 3 and st["general_segments"] == 32, st
    for calls in ([("sum", 0), ("count", 0), ("max", 0)], [(f, 0) for f in ALL6], [("count", 0)]):
        run_both(sh, sd, calls, iv, tmin, tmax, f"neighbouring heads {before_x} s before X {calls}")
    sh.close()


def test_series_offset_by_whole_segments():
    """Equal segment counts, but half the series start two segments later: segment index j then covers different times
    in different series.  Values are low-entropy on [2000 s, 3000 s) only, so the length-sorted lane groups of index 0
    (late series) and index 2 (early series) both cover that range with the same rank -- the same folded-matrix column."""
    rng = np.random.default_rng(6)

    def values(s, t):
        rel = (t - T0) // SEC
        calm = (rel >= 2000) & (rel < 3000)
        noisy = 100.0 + np.floor(rng.random(t.size) * 2.0**40) / 2.0**40
        return np.where(calm, 100.0 + (rel % 4) * 0.25, noisy)

    series = _grid(64, 3, 1000, values, start=lambda s: (2000 * SEC if s % 2 else 0))
    sh, sd = _open(series)
    tmax = T0 + 4999 * SEC
    for calls in ([("sum", 0), ("count", 0), ("max", 0)], [(f, 0) for f in ALL6]):
        run_both(sh, sd, calls, 60 * SEC, T0, tmax, f"offset {calls}")
    run_both(sh, sd, [("sum", 0), ("count", 0)], 60 * SEC, T0 + 2000 * SEC, T0 + 2999 * SEC, "offset, one range")
    sh.close()


def test_selector_ties_at_segment_boundaries():
    """Values from a tiny set, so the extreme of a window that crosses a segment boundary is tied between its two parts:
    the earlier time must win, as in the ordered stitch."""
    rng = np.random.default_rng(7)
    series = _grid(70, 4, 500, lambda s, t: 100.0 + rng.integers(0, 3, t.size) * 0.5)
    sh, sd = _open(series)
    tmax = T0 + 1999 * SEC
    for iv in (60 * SEC, 7 * SEC, 1000 * SEC):
        for f in ALL6:
            run_both(sh, sd, [(f, 0)], iv, T0, tmax, f"boundary ties {f} iv={iv}")
        run_both(sh, sd, [(f, 0) for f in ALL6], iv, T0, tmax, f"boundary ties multi iv={iv}")
    run_both(sh, sd, [("min", 0), ("last", 0), ("count", 0)], 60 * SEC, T0 + 250 * SEC + 3, T0 + 1750 * SEC, "boundary ties cut")
    sh.close()


@pytest.mark.parametrize("chunk", ["32", "7"])
def test_multi_chunk_plans_fold_edges(monkeypatch, chunk):
    """OGPU_CHUNK_SERIES: the folded matrix (lane-group, tail and stitched-edge columns) is filled and merged once per chunk."""
    monkeypatch.setenv("OGPU_CHUNK_SERIES", chunk)
    series = _grid(100, 3, 1000, _rng_values(8), jitter=lambda s, g: s == 41 and g == 1)
    sh, sd = _open(series)
    tmax = T0 + 2999 * SEC
    for calls in ([("sum", 0), ("count", 0), ("max", 0)], [(f, 0) for f in ALL6]):
        run_both(sh, sd, calls, 60 * SEC, T0, tmax, f"chunks {chunk} {calls}")
    run_both(sh, sd, [("sum", 0), ("min", 0)], 45 * SEC, T0 + 100 * SEC + 1, T0 + 2100 * SEC, f"chunks {chunk} cut")
    sh.close()
