"""CPU model of a whole-shard downsample (og_downsample_shard), built only from the oracle and numpy: nothing here imports the
library's Python layer beyond the ctypes structs and constants the oracle itself takes.

  1. per source field, the oracle's per-series window aggregates (oracle.scan, GROUP_PER_SERIES) for its type's calls;
     string fields, which the oracle does not decode, are counted from the validity the test wrote into their pages
  2. a series keeps a window where any output cell is non-null (the union row rule); the row time is the window start
  3. the kept rows of a series are cut into 1000-row segments
  4. pages come from the oracle's encoders, with the validity of each cell (bitmaps where a segment has null cells)
"""
import numpy as np

import oracle
from opengemini_b200 import _lib as L

ROWS = 1000
FUNC = {"count": L.AGG_COUNT, "sum": L.AGG_SUM, "min": L.AGG_MIN, "max": L.AGG_MAX, "first": L.AGG_FIRST, "last": L.AGG_LAST}


def schema(fields, ops):
    """fields: [(name, type)] in shard order; ops: {type: [call, ...]} -> [(out name, out type, field index, call)] by name."""
    out = []
    for i, (name, typ) in enumerate(fields):
        for f in ops.get(typ, []):
            out.append((f"{f}_{name}", L.TYPE_INT if f == "count" else typ, i, f))
    return sorted(out, key=lambda c: c[0])


def oracle_cells(desc, field, calls, interval, tmin, tmax):
    """The oracle's dense per-series record for `calls` over one field: grid (start, interval, n_buckets), {call: (u64, valid)}."""
    ca = (L.Call * len(calls))(*[(FUNC[f], field) for f in calls])
    qd = L.QueryDesc(interval, 0, tmin, tmax, 1, len(calls), ca, 0, None, L.GROUP_PER_SERIES, desc.n_series, None, 0, 0)
    r = oracle.scan(desc, qd, threads=1)
    return (r["start"], r["interval"], r["n_buckets"]), {f: (r["cols"][k]["values"].view(np.uint64), r["cols"][k]["valid"].astype(bool))
                                                         for k, f in enumerate(calls)}


def string_counts(series_rows, grid, tmin, tmax):
    """count() of a string field from its rows: series_rows = [(times, valid)] per series."""
    start, interval, nb = grid
    cnt = np.zeros(len(series_rows) * nb, np.int64)
    for s, (t, ok) in enumerate(series_rows):
        m = ok & (t >= tmin) & (t <= tmax)
        np.add.at(cnt, s * nb + (t[m] - start) // interval, 1)
    return cnt.view(np.uint64), cnt > 0


def expected(columns, cells, grid, n_series):
    """columns: schema(...); cells: {(field index, call): (u64 [n_series * nb], valid)} -> what the downsampled shard holds."""
    start, interval, nb = grid
    keep = np.zeros((n_series, nb), bool)
    for _n, _t, fi, f in columns:
        keep |= cells[(fi, f)][1].reshape(n_series, nb)
    ssb, seg_times, seg_win, rows = [0], [], [], 0
    for s in range(n_series):
        w = np.nonzero(keep[s])[0]
        rows += w.size
        for a in range(0, w.size, ROWS):
            seg_win.append((s, w[a:a + ROWS]))
            seg_times.append(start + w[a:a + ROWS].astype(np.int64) * interval)
        ssb.append(len(seg_win))
    cols = []
    for name, typ, fi, f in columns:
        v, ok = cells[(fi, f)]
        segs = []
        for s, w in seg_win:
            sv, sok = v[s * nb + w].copy(), ok[s * nb + w]
            sv[~sok] = 0
            segs.append((sv, sok))
        cols.append((name, typ, segs))
    return dict(ssb=np.array(ssb, np.uint32), rows=rows, seg_times=seg_times, cols=cols)


def cell_array(typ, u64):
    """Model cells in the form the oracle's encoders take."""
    if typ == L.TYPE_FLOAT:
        return u64.view(np.float64)
    if typ == L.TYPE_BOOL:
        return (u64 != 0).astype(np.uint8)
    return u64.view(np.int64)


def pages(model):
    """The oracle's page bytes for every output column and segment, then the time column's."""
    out = []
    for _name, typ, segs in model["cols"]:
        out.append([oracle.field_page_encode(typ, cell_array(typ, v), ok.astype(np.uint8)) for v, ok in segs])
    out.append([oracle.time_page_encode(t) for t in model["seg_times"]])
    return out
