"""The reference's per-query read of a shard's file set, restated in Python (test infrastructure only).

Structured as the reference reads it, so that the records handed to the aggregate cursor are cut where the reference cuts them:

  1. every file is sliced to the query range and filtered per file (Location.ReadData with filterOpts, engine/file_cursor.go:317-321:
     FilterByTime / FilterByField, engine/immutable/reader.go:754-974);
  2. the out-of-order files are folded newest first, per series: acc = MergeRecordLimitRows(acc, older, 0, 0, rows(acc) + rows(older))
     (engine/agg_tagset_cursor.go:411-436,515-535);
  3. each ordered record (one segment) of a series is merged with what is left of the folded out-of-order record by mergeData ->
     MergeRecordByMaxTimeOfOldRec at ChunkSizeNum rows (engine/file_cursor.go:292-348, engine/iterators_helper.go:484-520,
     lib/record/record.go:843-880); what is left after the last ordered record is cut into ChunkSizeNum-row records (cutRecord,
     iterators_helper.go:204-213);
  4. the records go to the existing CPU oracle (tests/oracle.py -> oracle/scan.cpp: aggregate cursor and tagset merge) as the
     segments of one ordered shard, one record per segment, with the WHERE already applied.

The record merge functions restate lib/record/record.go:363-505,610-880 (ascending only).  A Record is a dict:
{"schema": [(name, type)...] sorted by name (time excluded), "cols": {name: [value or None per row]}, "times": [int]}.
"""
import numpy as np

import oracle
from opengemini_b200 import _lib as L
from opengemini_b200.cursor import Shard

CHUNK_SIZE_NUM = 1024  # ChunkSizeNum default (og_query_desc.chunk_size <= 0)


# ---------------------------------------------------------------- lib/record/record.go
def rec_new(schema=()):
    return {"schema": list(schema), "cols": {n: [] for n, _t in schema}, "times": []}


def rows(r):
    return len(r["times"])


def _schema_union(new, old):  # mergeRecordSchema :438-466 (the newer file's type where both hold a name)
    out = dict(old["schema"])
    out.update(dict(new["schema"]))
    return sorted(out.items())


def _ensure(rec, schema):
    n = rows(rec)
    for name, ty in schema:
        if name not in rec["cols"]:
            rec["cols"][name] = [None] * n
    rec["schema"] = sorted(dict(rec["schema"] + list(schema)).items())


def append_rec(rec, src, start, end):  # AppendRec: columns the source lacks are padded with nulls (PadColVal)
    n = end - start
    if n <= 0:
        return
    _ensure(rec, src["schema"])
    for name, _t in rec["schema"]:
        rec["cols"][name] += src["cols"][name][start:end] if name in src["cols"] else [None] * n
    rec["times"] += src["times"][start:end]


def merge_rec_row(rec, new, old, i_new, i_old):  # mergeRecRow :468-505
    _ensure(rec, _schema_union(new, old))
    for name, _t in rec["schema"]:
        nv = new["cols"][name][i_new] if name in new["cols"] else None
        ov = old["cols"][name][i_old] if name in old["cols"] else None
        rec["cols"][name].append(nv if nv is not None else ov)
    rec["times"].append(new["times"][i_new])


def _non_overlap(rec, new, old, new_pos, old_pos, new_rows, old_rows, limit):  # mergeRecordNonOverlap :363-436: old rows first
    _ensure(rec, _schema_union(new, old))
    if old_rows - old_pos < limit:
        old_end = old_rows
        limit -= old_rows - old_pos
        new_end = new_rows if new_rows - new_pos <= limit else new_pos + limit
    else:
        old_end = old_pos + limit
        new_end = new_pos
    append_rec(rec, old, old_pos, old_end)
    append_rec(rec, new, new_pos, new_end)
    return new_end, old_end


def start_index(times, start_pos, t):  # GetTimeRangeStartIndex lib/record/utils.go:89-103
    lo, hi = start_pos, len(times) - 1
    while lo <= hi:
        mid = (lo + hi) // 2
        if times[mid] == t:
            return mid
        if times[mid] < t:
            lo = mid + 1
        else:
            hi = mid - 1
    return lo


def end_index(times, start_pos, t):  # GetTimeRangeEndIndex lib/record/utils.go:137-153
    lo, hi = start_pos, len(times) - 1
    while lo <= hi:
        mid = (lo + hi) // 2
        if times[mid] == t:
            return mid
        if times[mid] < t:
            lo = mid + 1
        else:
            hi = mid - 1
    return hi


def _append_recs(rec, new, old, ns, ne, os_, oe, nt, ot, limit):  # appendRecs :610-668 (ascending)
    while ns < ne and os_ < oe:
        if ot[os_] < nt[ns]:
            append_rec(rec, old, os_, os_ + 1); os_ += 1
        elif nt[ns] < ot[os_]:
            append_rec(rec, new, ns, ns + 1); ns += 1
        else:
            merge_rec_row(rec, new, old, ns, os_); ns += 1; os_ += 1
        limit -= 1
        if limit == 0:
            return 0, ns, os_
    if ns < ne:
        if ne - ns >= limit:
            append_rec(rec, new, ns, ns + limit)
            return 0, ns + limit, os_
        append_rec(rec, new, ns, ne)
        limit -= ne - ns
    elif os_ < oe:
        if oe - os_ >= limit:
            append_rec(rec, old, os_, os_ + limit)
            return 0, ns, os_ + limit
        append_rec(rec, old, os_, oe)
        limit -= oe - os_
    return limit, ne, oe


def _overlap_impl(rec, new, old, ns, ne, os_, oe, nt, ot, new_pos, old_pos, new_rows, old_rows, limit):  # mergeRecordOverlapImpl :670-719
    ne, oe = min(ne, new_rows), min(oe, old_rows)
    if os_ == old_pos:
        cur = ns - new_pos
        if cur >= limit:
            append_rec(rec, new, new_pos, new_pos + limit)
            return new_pos + limit, old_pos
        append_rec(rec, new, new_pos, ns)
        limit -= cur
    else:
        cur = os_ - old_pos
        if cur >= limit:
            append_rec(rec, old, old_pos, old_pos + limit)
            return new_pos, old_pos + limit
        append_rec(rec, old, old_pos, os_)
        limit -= cur
    limit, new_end, old_end = _append_recs(rec, new, old, ns, ne, os_, oe, nt, ot, limit)
    if limit == 0:
        return new_end, old_end
    if old_end == old_rows:
        if new_rows - new_end >= limit:
            append_rec(rec, new, new_end, new_end + limit)
            return new_end + limit, old_end
        append_rec(rec, new, new_end, new_rows)
        return new_rows, old_rows
    if old_rows - old_end >= limit:
        append_rec(rec, old, old_end, old_end + limit)
        return new_end, old_end + limit
    append_rec(rec, old, old_end, old_rows)
    return new_rows, old_rows


def _overlap(rec, new, old, nt, ot, new_pos, old_pos, new_rows, old_rows, limit):  # mergeRecordOverlap :721-760
    _ensure(rec, _schema_union(new, old))
    si = start_index
    if nt[new_pos] < ot[old_pos]:
        if nt[new_rows - 1] <= ot[old_rows - 1]:
            return _overlap_impl(rec, new, old, si(nt, new_pos, ot[old_pos]), new_rows, old_pos, si(ot, old_pos, nt[new_rows - 1]) + 1,
                                 nt, ot, new_pos, old_pos, new_rows, old_rows, limit)
        return _overlap_impl(rec, new, old, si(nt, new_pos, ot[old_pos]), si(nt, new_pos, ot[old_rows - 1]) + 1, old_pos, old_rows,
                             nt, ot, new_pos, old_pos, new_rows, old_rows, limit)
    if nt[new_rows - 1] <= ot[old_rows - 1]:
        return _overlap_impl(rec, new, old, new_pos, new_rows, si(ot, old_pos, nt[new_pos]), si(ot, old_pos, nt[new_rows - 1] + 1),
                             nt, ot, new_pos, old_pos, new_rows, old_rows, limit)
    return _overlap_impl(rec, new, old, new_pos, si(nt, new_pos, ot[old_rows - 1]) + 1, si(ot, old_pos, nt[new_pos]), old_rows,
                         nt, ot, new_pos, old_pos, new_rows, old_rows, limit)


def merge_record_limit_rows(rec, new, old, new_pos, old_pos, limit):  # MergeRecordLimitRows :847-862
    nt, ot = new["times"], old["times"]
    if nt[new_pos] > ot[-1]:
        return _non_overlap(rec, new, old, new_pos, old_pos, len(nt), len(ot), limit)
    if nt[-1] < ot[old_pos]:
        old_end, new_end = _non_overlap(rec, old, new, old_pos, new_pos, len(ot), len(nt), limit)
        return new_end, old_end
    return _overlap(rec, new, old, nt, ot, new_pos, old_pos, len(nt), len(ot), limit)


def merge_record(rec, new, old):  # MergeRecord :838-840
    return merge_record_limit_rows(rec, new, old, 0, 0, rows(new) + rows(old))


def merge_record_by_max_time_of_old_rec(rec, new, old, new_pos, old_pos, limit):  # MergeRecordByMaxTimeOfOldRec :880-900 (ascending)
    nt, ot = new["times"], old["times"]
    if nt[new_pos] > ot[-1]:
        append_rec(rec, old, old_pos, len(ot))
        return new_pos, len(ot)
    if nt[-1] < ot[old_pos]:
        old_end, new_end = _non_overlap(rec, old, new, old_pos, new_pos, len(ot), len(nt), limit)
        return new_end, old_end
    e = end_index(nt, new_pos, ot[-1])
    return _overlap(rec, new, old, nt[:e + 1], ot, new_pos, old_pos, e + 1, len(ot), limit)


# ---------------------------------------------------------------- engine/iterators_helper.go
class RecordIter:  # recordIter :180-213
    def __init__(self, rec=None):
        self.rec, self.pos = rec, 0

    def remain(self):
        return self.rec is not None and self.pos < rows(self.rec)

    def cut(self, max_row):
        n = min(rows(self.rec) - self.pos, max_row)
        out = rec_new(self.rec["schema"])
        append_rec(out, self.rec, self.pos, self.pos + n)
        self.pos += n
        return out


def merge_data(new_it, base_it, max_row):  # mergeData :484-520 (ascending)
    if new_it.remain() and base_it.remain():
        out = rec_new()
        np_, op = merge_record_by_max_time_of_old_rec(out, new_it.rec, base_it.rec, new_it.pos, base_it.pos, max_row)
        new_it.pos, base_it.pos = np_, op
        return out
    if base_it.remain():
        return base_it.cut(max_row)
    if new_it.remain():
        return new_it.cut(max_row)
    return None


# ---------------------------------------------------------------- file-set read
def _filter_rows(rec, q, flt):
    """FilterByTime + FilterByField on one file's record (RPN of (column name, op, const) terms; a null cell fails its term)."""
    keep = []
    for i, t in enumerate(rec["times"]):
        if t < q["tmin"] or t > q["tmax"]:
            continue
        if flt:
            st = []
            for it in flt:
                if it in ("and", "or"):
                    b, a = st.pop(), st.pop()
                    st.append((a and b) if it == "and" else (a or b))
                    continue
                name, op, c = it
                v = rec["cols"].get(name, [None] * rows(rec))[i]
                if v is None:
                    st.append(False)
                    continue
                v = float(v) if isinstance(c, float) else v
                st.append({"<": v < c, "<=": v <= c, ">": v > c, ">=": v >= c, "=": v == c, "!=": v != c}[op])
            if not st[0]:
                continue
        keep.append(i)
    out = rec_new(rec["schema"])
    for i in keep:
        append_rec(out, rec, i, i + 1)
    return out


def read_files(files, q, flt=None, chunk=CHUNK_SIZE_NUM, seg_rows=1000):
    """files: [(series dict, out_of_order)] oldest first; series dict = {sid: {"times": int64[], "cols": {name: (type, values, valid)}}}
    (the layout of tests/test_gpu_out_of_order.py).  Returns {sid: [records in the order the aggregate cursor receives them]}."""
    def records_of(s, cut):
        names = sorted(s["cols"])
        schema = [(n, s["cols"][n][0]) for n in names]
        t = s["times"].tolist()
        out = []
        for a in range(0, len(t), cut):
            b = min(a + cut, len(t))
            r = rec_new(schema)
            r["times"] = t[a:b]
            for n in names:
                _ty, v, ok = s["cols"][n]
                r["cols"][n] = [(v[k].item() if hasattr(v[k], "item") else v[k]) if ok[k] else None for k in range(a, b)]
            out.append(r)
        return out

    ooo_files = [f for f, ooo in files if ooo]
    ordered_files = [f for f, ooo in files if not ooo]
    acc = {}
    for f in reversed(ooo_files):  # newest first
        for sid, s in f.items():
            r = _filter_rows(records_of(s, max(1, s["times"].size))[0], q, flt) if s["times"].size else rec_new()
            if not rows(r):
                continue
            if sid not in acc:
                acc[sid] = r
            else:
                m = rec_new()
                merge_record_limit_rows(m, acc[sid], r, 0, 0, rows(acc[sid]) + rows(r))
                acc[sid] = m
    out = {}
    sids = sorted({sid for f, _ in files for sid in f})
    for sid in sids:
        mem = RecordIter(acc.get(sid))
        recs = []
        for f in ordered_files:
            if sid not in f:
                continue
            for seg in records_of(f[sid], seg_rows):  # Location.ReadData: one segment per record
                seg = _filter_rows(seg, q, flt)
                if not rows(seg):
                    continue
                base = RecordIter(seg)
                while base.remain():
                    recs.append(merge_data(mem, base, chunk))
        while mem.remain():
            recs.append(merge_data(mem, RecordIter(), chunk))
        out[sid] = [r for r in recs if r is not None and rows(r)]
    return out


def scan_aggregate_files(files, query, flt=None, seg_rows=1000):
    """Aggregate the file set as the reference does: read_files, then the CPU oracle's aggregate cursor + tagset merge over one
    ordered shard whose segments are those records.  `query` is the AggQuery whose descriptor (without its WHERE) is scanned;
    `flt` is the WHERE as (column name, op, const) RPN terms, applied per file; `seg_rows` is the segment length of the ordered files
    (each of their segments is one record)."""
    d = query.desc
    recs = read_files(files, {"tmin": d.tmin, "tmax": d.tmax}, flt, chunk=d.chunk_size if d.chunk_size > 0 else CHUNK_SIZE_NUM, seg_rows=seg_rows)
    names = sorted({n for f, _ in files for s in f.values() for n in s["cols"]})
    types = {n: t for f, _ in files for s in f.values() for n, (t, _v, _k) in s["cols"].items()}
    blob, pos = [], 0
    po = {n: [] for n in names}; pl = {n: [] for n in names}
    tpo, tpl, tmin, tmax, ssb, sid_list = [], [], [], [], [0], []

    def put(page):
        nonlocal pos
        blob.append(np.asarray(page, np.uint8)); off = pos; pos += len(page)
        return off, len(page)

    for sid in sorted(recs):
        for r in recs[sid]:
            for n in names:
                col = r["cols"].get(n)
                if col is None or all(v is None for v in col):
                    po[n].append(0); pl[n].append(0); continue
                ty = types[n]
                dt = np.uint8 if ty == L.TYPE_BOOL else np.float64 if ty == L.TYPE_FLOAT else np.int64
                cells = np.array([0 if v is None else v for v in col], dt)
                ok = np.array([v is not None for v in col], np.uint8)
                o, ln = put(oracle.field_page_encode(ty, cells, ok))
                po[n].append(o); pl[n].append(ln)
            t = np.array(r["times"], np.int64)
            o, ln = put(oracle.time_page_encode(t))
            tpo.append(o); tpl.append(ln); tmin.append(int(t[0])); tmax.append(int(t[-1]))
        ssb.append(len(tmin)); sid_list.append(sid)
    if tmin:  # the interval record spans the files' time range (FileInfo.MinTime/MaxTime), whatever the WHERE removed
        tmin[0] = min(tmin[0], min(int(s["times"][0]) for f, _ in files for s in f.values() if s["times"].size))
        tmax[-1] = max(tmax[-1], max(int(s["times"][-1]) for f, _ in files for s in f.values() if s["times"].size))
    data = np.concatenate(blob) if blob else np.zeros(1, np.uint8)
    desc = Shard.desc(data, sid_list, ssb, tmin, tmax, [(n, types[n], po[n], pl[n]) for n in names], tpo, tpl)
    saved = (d.n_filter, d.filter)
    d.n_filter = 0
    try:
        return oracle.scan(desc, d, threads=1), sid_list
    finally:
        d.n_filter, d.filter = saved
