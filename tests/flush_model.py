"""CPU model of og_shard_append_rows, built from numpy and the oracle's encoders: the two files the reference's memtable flush writes
for one batch of rows.

  1. per series, sort and deduplicate (WriteChunk.SortRecord -> ColumnSortHelper.Sort, lib/record/column_sort.go:42-97): rows
     sorted stably by time; for a run of equal times each column takes the last non-null value in arrival order, a null never
     replaces a value (replace, :100-107)
  2. split at the series' last time in the shard (SplitRecordByTime, engine/mutable/ts_table.go:242-290): t > last ordered,
     t <= last out of order; a column with no non-null value in a part is left out of that part (:276-286), also when every row
     falls into one part, where the reference hands the record on unchanged and keeps such a column (:243-248; DESIGN.md
     "Deviations")
  3. each part is one series of a file; file_desc cuts it into 1000-row segments from its first row (WriteData), every kept
     column with a page in each, pages from compact_model.encode_field (raw page where Gorilla refuses a float segment)

A batch is {sid: {"times", "cols": {name: (type, values per row, valid per row)}}}, the form test_gpu_out_of_order._series builds.
"""
import numpy as np

import compact_model as cm
import oracle
from opengemini_b200 import Shard
from opengemini_b200 import _lib as L

INT64_MIN = -(1 << 63)


def _dtype(typ):
    return np.uint8 if typ == L.TYPE_BOOL else np.float64 if typ == L.TYPE_FLOAT else np.int64


def sort_dedup(times, cols):
    """One series' record in arrival order -> (times ascending and unique, {name: (type, values, valid)}) by the sort rule."""
    times = np.asarray(times, np.int64)
    order = np.argsort(times, kind="stable")
    ts = times[order]
    uniq, start = np.unique(ts, return_index=True)
    out = {}
    for name, (typ, v, ok) in cols.items():
        v, ok = np.asarray(v)[order], np.asarray(ok, bool)[order]
        idx = np.where(ok, np.arange(ts.size), -1)
        last = np.maximum.reduceat(idx, start) if ts.size else np.zeros(0, np.int64)  # last valid row of each run, -1 when none
        has = last >= 0
        vals = np.zeros(uniq.size, _dtype(typ))
        vals[has] = v[last[has]]
        out[name] = (typ, vals, has)
    return uniq, out


def split(times, cols, last):
    """-> (ordered part, out-of-order part), each None or (times, cols) with the columns that hold a value in the part."""
    parts = []
    for sel in (times > last, times <= last):
        if not sel.any():
            parts.append(None)
            continue
        kept = {n: (t, v[sel], ok[sel]) for n, (t, v, ok) in cols.items() if ok[sel].any()}
        parts.append((times[sel], kept))
    return parts[0], parts[1]


def flush(batch, last_of_sid=None):
    """-> (ordered file, out-of-order file, rows_replaced): {sid: {"times", "cols"}} each, series without rows in a part left out.
    last_of_sid: the shard's last time per sid (a sid it lacks: INT64_MIN)."""
    last_of_sid = last_of_sid or {}
    ordered, ooo, replaced = {}, {}, 0
    for sid in sorted(batch):
        s = batch[sid]
        t, cols = sort_dedup(s["times"], s["cols"])
        replaced += len(s["times"]) - t.size
        o, x = split(t, cols, last_of_sid.get(sid, INT64_MIN))
        if o is not None:
            ordered[sid] = dict(times=o[0], cols=o[1])
        if x is not None:
            ooo[sid] = dict(times=x[0], cols=x[1])
    return ordered, ooo, replaced


def files(batch, last_of_sid=None):
    """the flush as og_shard_append_files takes it: [(file, out_of_order)], ordered first, empty files left out"""
    o, x, _ = flush(batch, last_of_sid)
    return [(f, ooo) for f, ooo in ((o, False), (x, True)) if f]


def file_pages(series, seg_rows=1000):
    """{sid: {"times", "cols"}} -> (names, types, [(sid, [(tmin, tmax, {name: page}, time page)] per segment)])"""
    names = sorted({n for s in series.values() for n in s["cols"]})
    types = {n: t for s in series.values() for n, (t, _v, _k) in s["cols"].items()}
    out = []
    for sid in sorted(series):
        s = series[sid]
        t = s["times"]
        segs = []
        for a in range(0, t.size, seg_rows):
            b = min(a + seg_rows, t.size)
            pages = {n: cm.encode_field(types[n], np.ascontiguousarray(v[a:b]), np.asarray(ok[a:b], bool))
                     for n, (_ty, v, ok) in s["cols"].items()}
            segs.append((int(t[a]), int(t[b - 1]), pages, oracle.time_page_encode(t[a:b])))
        out.append((sid, segs))
    return names, types, out


def file_desc(series, seg_rows=1000):
    """One file as a Shard.desc: pages from the encoders of the model, back to back."""
    names, types, segs = file_pages(series, seg_rows)
    blob, pos = [], 0
    po = {n: [] for n in names}; pl = {n: [] for n in names}
    tpo, tpl, tmin, tmax, ssb, sids = [], [], [], [], [0], []
    for sid, ss in segs:
        for lo, hi, pages, tp in ss:
            for n in names:
                p = pages.get(n)
                if p is None:
                    po[n].append(0); pl[n].append(0); continue
                blob.append(np.asarray(p, np.uint8)); po[n].append(pos); pl[n].append(len(p)); pos += len(p)
            blob.append(np.asarray(tp, np.uint8)); tpo.append(pos); tpl.append(len(tp)); pos += len(tp)
            tmin.append(lo); tmax.append(hi)
        ssb.append(len(tmin)); sids.append(sid)
    data = np.concatenate(blob) if blob else np.zeros(1, np.uint8)
    return Shard.desc(data, sids, ssb, tmin, tmax, [(n, types[n], po[n], pl[n]) for n in names], tpo, tpl)


def last_times(ex):
    """{sid: last time} of a shard's export (the latest seg_tmax of each series)"""
    ssb = ex["series_seg_begin"]
    return {int(sid): int(ex["seg_tmax"][ssb[i + 1] - 1]) for i, sid in enumerate(ex["sids"].tolist()) if ssb[i + 1] > ssb[i]}
