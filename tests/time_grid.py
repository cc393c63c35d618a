"""Plain-Python model of the query's time geometry, in unbounded ints: which rows of a shard are in range, which window each
row belongs to, and which bucket of the dense interval record a window's partial lands in.

It restates the reference from its definitions and shares no code with oracle/ or the library:
- window(): ProcessorOptions.Window (influxql select.go), clamped at MinTime/MaxTime;
- grid(): TimeWindowsInit over the query range intersected with the shard's rows (start, interval time, bucket count);
- placement: GetIndex of the time of the window's first row, |t - start| // interval, dropped past the last bucket.
On an unclamped grid every row of a window has the same GetIndex; near the int64 limits they may differ, and the model
follows the first row, as the partials of count, sum and multi-call queries do.
"""
import math
from dataclasses import dataclass

MIN_TIME = -2**63 + 2
MAX_TIME = 2**63 - 2


def window(interval, offset, tmin, tmax, t):
    """(start, end) of the window that holds t."""
    if interval == 0:
        return tmin, tmax + 1
    t -= offset
    dt = t % interval  # floor modulo: Window()'s truncated remainder plus its correction of negative values
    s = MIN_TIME if MIN_TIME + dt >= t else t - dt
    d2 = interval - dt
    e = MAX_TIME if MAX_TIME - d2 <= t else t + d2
    return s + offset, e + offset


@dataclass
class Grid:
    start: int      # what the dense record reports: 0 without an interval
    interval: int   # interval time of the first window (the record's bucket width)
    n_buckets: int
    tmin: int       # the query range after the MinTime/MaxTime clamp
    tmax: int
    has_interval: bool
    clamped: bool   # the window of the first or last row in range is clamped at MIN_TIME/MAX_TIME


def grid(interval, offset, tmin, tmax, data_tmin, data_tmax, query_grid=False):
    """TimeWindowsInit over [max(tmin, data_tmin), min(tmax, data_tmax)]; query_grid: the query range itself (OG_Q_QUERY_GRID)."""
    tmin, tmax = max(tmin, MIN_TIME), min(tmax, MAX_TIME)
    gmin, gmax = max(tmin, data_tmin), min(tmax, data_tmax)
    overlap = gmin <= gmax
    if not overlap:
        gmin = gmax = tmin
    if query_grid:
        gmin, gmax, overlap = tmin, tmax, True
    if interval == 0:
        return Grid(0, gmax + 1 - gmin, 1, tmin, tmax, False, False)
    s0, e0 = window(interval, offset, tmin, tmax, gmin)
    s1, e1 = window(interval, offset, tmin, tmax, gmax + 1)
    iv = e0 - s0
    sl, el = window(interval, offset, tmin, tmax, gmax)
    clamped = overlap and (e0 - s0 != interval or el - sl != interval)
    return Grid(s0, iv, (e1 - s0) // iv, tmin, tmax, True, clamped)


def place(times, g, interval, offset):
    """Bucket of every row of one series (times ascending): -1 for rows out of range or dropped past the last bucket."""
    out = [-1] * len(times)
    cur = None
    first = None
    for i, t in enumerate(times):
        if not (g.tmin <= t <= g.tmax):
            continue
        if not g.has_interval:
            out[i] = 0
            continue
        w = window(interval, offset, g.tmin, g.tmax, t)
        if w != cur:
            cur, first = w, t
        b = abs(first - g.start) // g.interval
        out[i] = b if b < g.n_buckets else -1
    return out


def bucket_rows(series, g, interval, offset):
    """series: list of ascending time lists.  Returns {bucket: [(series, row), ...]} of the rows the query aggregates."""
    rows = {}
    for s, times in enumerate(series):
        for r, b in enumerate(place(times, g, interval, offset)):
            if b >= 0:
                rows.setdefault(b, []).append((s, r))
    return rows


def expected(rows, times, values, valid=None):
    """Per-bucket reference answers of one float or int column over one group (all series).
    times[s][r], values[s][r]; valid[s][r] (None: every row valid).  Returns {bucket: dict(count, sum, min, max, first,
    last)}; min/max carry (time, value) with the earliest time among equal extremes, first/last (time, value) with the
    larger value on equal times."""
    out = {}
    for b, rs in rows.items():
        vs = [(times[s][r], values[s][r]) for s, r in rs if valid is None or valid[s][r]]
        if not vs:
            continue
        fmin = min(vs, key=lambda tv: (tv[1], tv[0]))
        fmax = max(vs, key=lambda tv: (tv[1], -tv[0]))
        t_first = min(t for t, _ in vs)
        t_last = max(t for t, _ in vs)
        out[b] = dict(count=len(vs), sum=math.fsum(v for _, v in vs) if isinstance(vs[0][1], float) else sum(v for _, v in vs),
                      min=fmin, max=fmax,
                      first=(t_first, max(v for t, v in vs if t == t_first)),
                      last=(t_last, max(v for t, v in vs if t == t_last)))
    return out
