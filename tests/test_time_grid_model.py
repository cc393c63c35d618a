"""The time-geometry model (time_grid.py) against the CPU oracle: window bounds, the grid of the dense record (start,
interval, bucket count) and the rows of every bucket, on cadences, intervals, offsets and range ends away from the
one-second grid, and near the int64 time limits, where Window() clamps the first or last window.  CPU only."""
import ctypes as C
import math

import numpy as np
import pytest

import oracle
import time_grid as tg
from opengemini_b200 import _lib as L

SEC = 1_000_000_000
DAY = 86_400 * SEC
T0 = 1_700_000_000_000_000_000


def host_shard(series, rows_per_seg=1000, seed=0):
    """series: list of (t0, dt, rows).  One float column of distinct values; pages from the oracle's encoders."""
    rng = np.random.default_rng(seed)
    pages, tpages, tmins, tmaxs, ssb = [], [], [], [], [0]
    times, values = [], []
    total = sum(n for _, _, n in series)
    pool = 100.0 + rng.permutation(total).astype(np.float64) / 1024.0
    k = 0
    for t0, dt, n in series:
        t = [t0 + i * dt for i in range(n)]
        v = pool[k:k + n]; k += n
        times.append(t); values.append([float(x) for x in v])
        for a in range(0, n, rows_per_seg):
            ts = np.array(t[a:a + rows_per_seg], np.int64)
            pages.append(oracle.field_page_encode(L.TYPE_FLOAT, v[a:a + rows_per_seg]))
            tpages.append(oracle.time_page_encode(ts)); tmins.append(int(ts[0])); tmaxs.append(int(ts[-1]))
        ssb.append(len(pages))
    blob, offs, lens, pos = [], [], [], 0
    for p in pages + tpages:
        offs.append(pos); lens.append(p.size); blob.append(p); pos += p.size
    nseg = len(pages)
    ex = dict(data=np.concatenate(blob), sids=np.arange(1, len(series) + 1, dtype=np.uint64),
              series_seg_begin=np.array(ssb, np.uint32), seg_tmin=np.array(tmins, np.int64), seg_tmax=np.array(tmaxs, np.int64),
              page_off=np.array([offs[:nseg], offs[nseg:]], np.uint64), page_len=np.array([lens[:nseg], lens[nseg:]], np.uint32),
              col_types=np.array([L.TYPE_FLOAT], np.int32))
    return oracle.shard_desc_from_export(ex), times, values


def query_desc(funcs, interval, offset, tmin, tmax):
    calls = (L.Call * len(funcs))()
    for i, f in enumerate(funcs):
        calls[i].func, calls[i].column = {"count": L.AGG_COUNT, "sum": L.AGG_SUM, "first": L.AGG_FIRST, "min": L.AGG_MIN}[f], 0
    d = L.QueryDesc()
    d.interval, d.offset, d.tmin, d.tmax, d.ascending = interval, offset, tmin, tmax, 1
    d.n_calls, d.calls, d.n_filter, d.group_mode, d.chunk_size = len(funcs), calls, 0, L.GROUP_ALL, 1024
    d._keep = calls
    return d


# name: (series [(t0, dt, rows)], interval, offset, tmin, tmax, clamped)
OPEN = (tg.MIN_TIME, tg.MAX_TIME)
CASES = {
    "1ns_cadence_1ns_interval": ([(T0, 1, 300)], 1, 0, *OPEN, False),
    "7ns_cadence_10ns_interval_offset1": ([(T0 + 3, 7, 500), (T0, 7, 500)], 10, 1, *OPEN, False),
    "3ns_cadence_10ns_interval": ([(T0, 3, 700)], 10, 0, *OPEN, False),
    "prime_cadence_dt_minus_1": ([(T0, 999_999_937, 400)], 999_999_936, 0, *OPEN, False),
    "prime_cadence_dt_plus_1": ([(T0, 999_999_937, 400)], 999_999_938, 5, *OPEN, False),
    "cadence_over_interval": ([(T0, 3 * SEC, 300)], SEC, 0, *OPEN, False),
    "365_days_over_1ns": ([(T0, 1, 2000)], 365 * DAY, 0, *OPEN, False),
    "offset_minus_two_intervals": ([(T0, 7, 900)], 60, -2 * 60 - 5, *OPEN, False),
    "offset_interval_plus_3": ([(T0, 7, 900)], 60, 63, *OPEN, False),
    "range_ends_off_rows": ([(T0, 7, 900)], 60, 0, T0 + 7 * 10 + 1, T0 + 7 * 800 - 1, False),
    "range_between_rows": ([(T0, 7, 900)], 60, 0, T0 + 7 * 10 + 1, T0 + 7 * 11 - 1, False),
    "range_one_row": ([(T0, 7, 900)], 60, 0, T0 + 7 * 10, T0 + 7 * 10, False),
    "no_interval": ([(T0, 7, 900), (T0 + 2, 7, 900)], 0, 0, *OPEN, False),
    "near_2_62": ([(2**62 - 1000, 1, 3000)], 7, 0, *OPEN, False),
    "near_minus_2_62": ([(-2**62 - 1000, 7, 3000)], 60, 3, *OPEN, False),
    # the last rows lie within one interval of MAX_TIME: Window() clamps the last window, one bucket short
    "last_window_clamped_at_max_time": ([(tg.MAX_TIME - 7 * 299, 7, 300)], 100, 0, *OPEN, True),
    # the first rows lie within one interval of MIN_TIME: the first window is clamped, the record's bucket width shrinks
    "first_window_clamped_at_min_time": ([(tg.MIN_TIME + 3, 7, 300)], 100, 0, *OPEN, True),
    # the first row on the first window boundary above MIN_TIME: nothing is clamped
    "first_row_on_the_first_boundary_above_min_time": ([(tg.MIN_TIME + (-tg.MIN_TIME) % 100, 7, 300)], 100, 0, *OPEN, False),
    # the last row ends the last whole window below MAX_TIME: only the (empty) window after it is clamped
    "last_row_just_below_the_last_boundary": ([(tg.MAX_TIME - tg.MAX_TIME % 100 - 1 - 7 * 299, 7, 300)], 100, 0, *OPEN, False),
}


@pytest.mark.parametrize("name", sorted(n for n, c in CASES.items() if c[1]))
def test_window_bounds(name):
    series, interval, offset, tmin, tmax, _ = CASES[name]
    probes = {tmin, tmax, tg.MIN_TIME, tg.MAX_TIME, -1, 0, 1}
    for t0, dt, n in series:
        for r in (0, 1, n // 2, n - 2, n - 1):
            t = t0 + r * dt
            probes |= {t - 1, t, t + 1}
    for t in sorted(probes):
        w = tg.window(interval, offset, tmin, tmax, t)
        # where t - offset or a bound leaves int64, Window()'s int64 arithmetic wraps: the model does not follow it there
        if tg.MIN_TIME <= t <= tg.MAX_TIME and all(-2**63 <= x < 2**63 for x in (t - offset, *w)):
            assert w == oracle.window(interval, offset, tmin, tmax, t), (name, t)


@pytest.mark.parametrize("name", sorted(CASES))
def test_grid_and_rows_per_bucket(name):
    series, interval, offset, tmin, tmax, clamped = CASES[name]
    sd, times, values = host_shard(series)
    data_tmin = min(t[0] for t in times)
    data_tmax = max(t[-1] for t in times)
    g = tg.grid(interval, offset, tmin, tmax, data_tmin, data_tmax)
    assert g.clamped == clamped, name
    rows = tg.bucket_rows(times, g, interval, offset)
    want = tg.expected(rows, times, values)
    for funcs in (["count"], ["sum"], ["count", "first", "sum"]):
        ref = oracle.scan(sd, query_desc(funcs, interval, offset, tmin, tmax))
        assert (ref["start"], ref["n_buckets"]) == (g.start, g.n_buckets), name
        assert ref["interval"] == (g.interval if g.has_interval else 0), name
        for k, f in enumerate(funcs):
            col = ref["cols"][k]
            valid = col["valid"].astype(bool)
            assert sorted(np.flatnonzero(valid).tolist()) == sorted(want), f"{name} {f}: buckets with rows"
            for b, w in want.items():
                v = col["values"][b]
                if f == "count":
                    assert int(v) == w["count"], (name, b)
                elif f == "sum":
                    got = float(np.uint64(v).view(np.float64))
                    assert math.isclose(got, w["sum"], rel_tol=1e-12, abs_tol=0.0), (name, b)
                else:
                    got = float(np.uint64(v).view(np.float64))
                    assert (int(col["times"][b]), got) == w["first"], (name, b)


def test_clamped_grids_lose_or_misplace_rows():
    """What the reference structure does on the two clamped grids (the library refuses both): at MAX_TIME the rows of the
    last window fall past the last bucket and are dropped; at MIN_TIME the record's bucket width is the clamped first
    window, so later windows land at GetIndex of their first row, several buckets apart."""
    series, interval, offset, tmin, tmax, _ = CASES["last_window_clamped_at_max_time"]
    sd, times, _v = host_shard(series)
    g = tg.grid(interval, offset, tmin, tmax, times[0][0], times[0][-1])
    rows = tg.bucket_rows(times, g, interval, offset)
    placed = sum(len(r) for r in rows.values())
    assert placed < len(times[0])
    ref = oracle.scan(sd, query_desc(["count"], interval, offset, tmin, tmax))
    assert int(ref["cols"][0]["values"][ref["cols"][0]["valid"].astype(bool)].sum()) == placed

    series, interval, offset, tmin, tmax, _ = CASES["first_window_clamped_at_min_time"]
    sd, times, _v = host_shard(series)
    g = tg.grid(interval, offset, tmin, tmax, times[0][0], times[0][-1])
    assert g.interval < interval
    rows = tg.bucket_rows(times, g, interval, offset)
    assert sum(len(r) for r in rows.values()) == len(times[0])
    assert max(rows) > len(rows)  # buckets between the windows stay empty
