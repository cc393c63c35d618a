"""og_shard_open_files: a shard's ordered and out-of-order files opened as one shard, overlapping rows merged on the device.

Files are built here from oracle-encoded pages.  The merge is checked against a plain-Python model of the reference's row rule
(lib/record/record.go:468-505 mergeRecRow: per series and time, each column takes the newest file's non-null value; every
out-of-order file is newer than every ordered one, later out-of-order files newer than earlier ones): og_decode_segment over the
merged shard must give the model's rows bit for bit, and queries on the merged shard must give what the oracle computes over a
single ordered file that holds the model's rows."""
import struct

import numpy as np
import pytest

import oracle
import oracle_files
import tssp_file
from opengemini_b200 import AggQuery, Shard
from opengemini_b200 import _lib as L

pytestmark = pytest.mark.gpu
T0, SEC = 1_700_000_000_000_000_000, 1_000_000_000
ALL6 = ["count", "sum", "min", "max", "first", "last"]
TYPE_STRING = 4


@pytest.fixture(scope="module", autouse=True)
def _device():
    Shard.init(0)


# ---------------------------------------------------------------- files and the model
def _series(times, cols):
    """cols: {name: (type, values per row, valid per row)}"""
    return dict(times=np.asarray(times, np.int64), cols=cols)


def _file_desc(series, seg_rows=1000):
    """A shard description of one file: {sid: _series(...)} -> Shard.desc, pages from the oracle's encoders."""
    names = sorted({n for s in series.values() for n in s["cols"]})
    types = {n: t for s in series.values() for n, (t, _v, _k) in s["cols"].items()}
    blob, pos = [], 0
    po = {n: [] for n in names}; pl = {n: [] for n in names}
    tpo, tpl, tmin, tmax, ssb, sids = [], [], [], [], [0], []

    def put(page):
        nonlocal pos
        blob.append(np.asarray(page, np.uint8)); off = pos; pos += len(page)
        return off, len(page)

    for sid in sorted(series):
        s = series[sid]
        t = s["times"]
        cuts = list(range(0, t.size, seg_rows)) + [t.size]
        for a, b in zip(cuts[:-1], cuts[1:]):
            for n in names:
                if n not in s["cols"]:
                    po[n].append(0); pl[n].append(0); continue
                ty, v, ok = s["cols"][n]
                if ty == TYPE_STRING:
                    o, ln = put(_string_page(np.asarray(ok[a:b], bool)))
                else:
                    o, ln = put(oracle.field_page_encode(ty, np.ascontiguousarray(v[a:b]), np.asarray(ok[a:b], np.uint8)))
                po[n].append(o); pl[n].append(ln)
            o, ln = put(oracle.time_page_encode(t[a:b]))
            tpo.append(o); tpl.append(ln); tmin.append(int(t[a])); tmax.append(int(t[b - 1]))
        ssb.append(len(tmin)); sids.append(sid)
    data = np.concatenate(blob) if blob else np.zeros(1, np.uint8)
    return Shard.desc(data, sids, ssb, tmin, tmax, [(n, types[n], po[n], pl[n]) for n in names], tpo, tpl)


def _string_page(valid, payload=b"\x10opaque-string-block-bytes"):
    rows = len(valid)
    nil = int(rows - valid.sum())
    if nil == 0:
        return np.frombuffer(bytes([34]) + struct.pack(">I", rows) + payload, np.uint8)
    if nil == rows:
        return np.frombuffer(bytes([44]) + struct.pack(">I", rows), np.uint8)
    bm = np.packbits(valid.astype(np.uint8), bitorder="little").tobytes()
    return np.frombuffer(bytes([TYPE_STRING]) + struct.pack(">I", len(bm)) + bm + struct.pack(">II", 0, nil) + payload, np.uint8)


def _model(files):
    """files: [(series dict, out_of_order)] oldest first -> merged {sid: _series} by the row rule."""
    order = sorted(range(len(files)), key=lambda i: (files[i][1], i))  # newness: ordered < out-of-order, then file sequence
    rows, types = {}, {}
    for i in order:
        for sid, s in files[i][0].items():
            r = rows.setdefault(sid, {})
            for k, t in enumerate(s["times"].tolist()):
                row = r.setdefault(t, {})
                for n, (ty, v, ok) in s["cols"].items():
                    types[n] = ty
                    if ok[k]:
                        row[n] = v[k]
    out = {}
    for sid, r in rows.items():
        ts = np.array(sorted(r), np.int64)
        cols = {}
        for n, ty in types.items():
            dt = np.uint8 if ty == L.TYPE_BOOL else np.float64 if ty == L.TYPE_FLOAT else np.int64
            v = np.zeros(ts.size, dt); ok = np.zeros(ts.size, bool)
            for k, t in enumerate(ts.tolist()):
                if n in r[t]:
                    v[k] = r[t][n]; ok[k] = True
            cols[n] = (ty, v, ok)
        out[sid] = _series(ts, cols)
    return out


def _rows_of(sh, sid_index):
    """og_decode_segment over every segment of one series of a shard, concatenated."""
    ex = sh.export()
    a, b = int(ex["series_seg_begin"][sid_index]), int(ex["series_seg_begin"][sid_index + 1])
    recs = [sh.decode_segment(g) for g in range(a, b)]
    times = np.concatenate([r["times"] for r in recs])
    cols = []
    for c in range(len(recs[0]["cols"])):
        valid = np.concatenate([r["cols"][c]["valid"] for r in recs])
        vals = np.concatenate([r["cols"][c]["values"] for r in recs])
        cols.append((valid, vals))
    return times, cols


def _check_rows(sh, model):
    ex = sh.export()
    assert ex["sids"].tolist() == sorted(model)
    names = sorted({n for s in model.values() for n in s["cols"]})
    for i, sid in enumerate(ex["sids"].tolist()):
        m = model[sid]
        times, cols = _rows_of(sh, i)
        assert np.array_equal(times, m["times"]), sid
        for c, n in enumerate(names):
            ty, v, ok = m["cols"][n]
            if ty == TYPE_STRING:
                continue
            valid, vals = cols[c]
            assert np.array_equal(valid, ok), (sid, n)
            want = v[ok]
            if ty == L.TYPE_BOOL:
                assert np.array_equal(vals.astype(np.uint8), want.astype(np.uint8)), (sid, n)
            else:
                assert np.array_equal(vals.view(np.uint64), want.view(np.uint64)), (sid, n)


def _random_files(seed, n_series=12, rows=2600, with_bool=True):
    """One ordered file (every series, 1 s cadence), then out-of-order files that rewrite and insert rows of some series,
    with nulls in the newer rows, columns present in only some files, and a series only the out-of-order files hold."""
    rng = np.random.default_rng(seed)

    def cols_for(n, present, null_p):
        c = {}
        if "fv" in present:
            c["fv"] = (L.TYPE_FLOAT, np.round(rng.normal(100, 20, n), 3) + rng.random(n) * 1e-6, rng.random(n) >= null_p)
        if "iv" in present:
            c["iv"] = (L.TYPE_INT, rng.integers(-1000, 1000, n).cumsum(), rng.random(n) >= null_p)
        if "bv" in present and with_bool:
            c["bv"] = (L.TYPE_BOOL, (rng.random(n) < 0.5).astype(np.uint8), rng.random(n) >= null_p)
        return c

    ordered = {}
    for s in range(n_series):
        t = T0 + np.arange(rows, dtype=np.int64) * SEC
        ordered[100 + s] = _series(t, cols_for(rows, {"fv", "iv", "bv"}, 0.05))
    ooo1, ooo2 = {}, {}
    for s in range(0, n_series, 3):  # every third series gets late writes
        k = int(rng.integers(50, 400))
        t = np.unique(T0 + rng.integers(-200, rows + 200, k) * SEC + np.where(rng.random(k) < 0.3, SEC // 2, 0))
        ooo1[100 + s] = _series(t, cols_for(t.size, {"fv", "iv"}, 0.2))          # no bool column in this file
        t2 = np.unique(np.concatenate([t[: t.size // 2], T0 + rng.integers(0, rows, 60) * SEC]))
        ooo2[100 + s] = _series(t2, cols_for(t2.size, {"fv", "bv"}, 0.3))          # overlaps ooo1 and the ordered file
    t = T0 + np.arange(0, 1500, 3, dtype=np.int64) * SEC
    ooo2[999] = _series(t, cols_for(t.size, {"fv", "iv", "bv"}, 0.1))             # only out-of-order files hold it
    return [(ordered, False), (ooo1, True), (ooo2, True)]


def _open(files, **kw):
    return Shard.open_files([(_file_desc(f, **kw), ooo) for f, ooo in files])


def _compare(sh, files, calls, iv, tmin, tmax, where=None, **kw):
    """Query the merged shard and scan_aggregate_files (tests/oracle_files.py: the reference's file-set read restated, then the CPU
    oracle's aggregate cursor) over the same files.  Bitwise, except float sums of groups that hold a series with out-of-order
    rows: those agree within 1e-12 relative (DESIGN.md "Deviations")."""
    names = sorted({n for f, _ in files for s_ in f.values() for n in s_["cols"]})
    flt = [(it if it in ("and", "or") else ("term", it[0], it[1], it[2])) for it in where] if where else None
    flt_named = [(it if it in ("and", "or") else (names[it[0]], it[1], it[2])) for it in where] if where else None
    q = AggQuery(sh, calls, iv, tmin, tmax, filter=flt, **kw).run()
    got = q.dense_host()
    ref, sids = oracle_files.scan_aggregate_files(files, q, flt_named)
    merged_sids = {sid for f, ooo in files if ooo for sid in f}
    is_merged = np.array([sid in merged_sids for sid in sids])
    group = kw.get("group", "all")
    if group == "series":
        g_merged = is_merged
    elif group == "map":
        g_merged = np.array([is_merged[np.asarray(kw["series_group"]) == g].any() for g in range(kw["n_groups"])])
    else:
        g_merged = np.array([is_merged.any()])
    cell_merged = np.repeat(g_merged, got["n_buckets"])
    for k, (f, c) in enumerate(calls):
        rv = ref["cols"][k]["valid"].astype(bool)
        assert np.array_equal(got["cols"][k]["valid"].astype(bool), rv), (f, c, iv, kw)
        g, r = got["cols"][k]["values"].view(np.uint64), ref["cols"][k]["values"]
        loose = rv & cell_merged if (f == "sum" and got["cols"][k]["type"] == L.TYPE_FLOAT) else np.zeros_like(rv)
        exact = rv & ~loose
        assert np.array_equal(g[exact], r[exact]), (f, c, iv, kw)
        gf, rf = g[loose].view(np.float64), r[loose].view(np.float64)
        assert np.all(np.abs(gf - rf) <= 1e-12 * np.maximum(1.0, np.abs(rf))), (f, c, iv, kw)
        if got["cols"][k]["times"] is not None and f in ("min", "max", "first", "last"):
            assert np.array_equal(got["cols"][k]["times"][rv], ref["cols"][k]["times"][rv]), (f, c, iv, kw)
    st = q.stats()
    q.close()
    return st


# ---------------------------------------------------------------- 1. one ordered file
def test_one_ordered_file_equals_og_shard_open():
    cols = [(L.TYPE_FLOAT, L.SYNTH_F_HI, 0), (L.TYPE_INT, L.SYNTH_INT_WALK, 30), (L.TYPE_BOOL, L.SYNTH_BOOL, 0)]
    base = Shard.synth(30, 2500, cols, t0=T0, dt=SEC, seed=5)
    desc = oracle.shard_desc_from_export(base.export())
    a = Shard.open_desc(desc)
    b = Shard.open_files([(desc, False)])
    ea, eb = a.export(), b.export()
    for k in ea:
        assert np.array_equal(ea[k], eb[k]), k
    assert a.info() == b.info()
    mi = b.merge_info()
    assert mi["n_files"] == 1 and mi["n_out_of_order_files"] == 0 and mi["series_merged"] == 0 and mi["segments_kept"] == ea["seg_tmin"].size
    assert a.merge_info()["n_files"] == 1 and a.merge_info()["segments_kept"] == 0
    for calls in ([("sum", 0), ("count", 0), ("max", 0)], [("min", 1), ("last", 2), ("sum", 1)]):
        for flags in (L.Q_STRICT_ORDER, 0):
            qa = AggQuery(a, calls, 60 * SEC, T0, T0 + 2499 * SEC, flags=flags).run()
            qb = AggQuery(b, calls, 60 * SEC, T0, T0 + 2499 * SEC, flags=flags).run()
            da, db = qa.dense_host(), qb.dense_host()
            for k in range(len(calls)):
                assert np.array_equal(da["cols"][k]["valid"], db["cols"][k]["valid"])
                assert np.array_equal(da["cols"][k]["values"].view(np.uint64), db["cols"][k]["values"].view(np.uint64))
            assert qa.stats()["path"] == qb.stats()["path"]
            qa.close(); qb.close()
    a.close(); b.close(); base.close()


# ---------------------------------------------------------------- 2. several ordered files
def _cut_by_segment(ex, n_files):
    """Ordered files cut by time from one exported shard: file j holds the j-th third of every series' segments."""
    nc = ex["col_types"].size
    ssb = ex["series_seg_begin"]
    descs = []
    for j in range(n_files):
        segs, fssb = [], [0]
        for s in range(ex["sids"].size):
            a, b = int(ssb[s]), int(ssb[s + 1])
            k = (b - a + n_files - 1) // n_files
            segs += list(range(a + j * k, min(b, a + (j + 1) * k)))
            fssb.append(len(segs))
        segs = np.array(segs, np.int64)
        descs.append(Shard.desc(ex["data"], ex["sids"], fssb, ex["seg_tmin"][segs], ex["seg_tmax"][segs],
                                [(f"f{c}", int(ex["col_types"][c]), ex["page_off"][c][segs], ex["page_len"][c][segs]) for c in range(nc)],
                                ex["page_off"][nc][segs], ex["page_len"][nc][segs]))
    return descs


def test_three_ordered_files_answer_like_one():
    cols = [(L.TYPE_FLOAT, L.SYNTH_F_HI, 0), (L.TYPE_INT, L.SYNTH_INT_WALK, 0)]
    one = Shard.synth(64, 6000, cols, t0=T0, dt=SEC, seed=11)
    descs = _cut_by_segment(one.export(), 3)
    three = Shard.open_files([(d, False) for d in descs])
    mi = three.merge_info()
    assert mi["n_files"] == 3 and mi["segments_rewritten_out"] == 0 and mi["segments_kept"] == one.info()["n_segments"]
    assert three.info()["n_rows"] == one.info()["n_rows"]
    tmax = T0 + 5999 * SEC
    for calls in ([("sum", 0), ("count", 0), ("max", 0)], [("sum", 0), ("count", 0)], [(f, 0) for f in ALL6], [("min", 1), ("sum", 1)]):
        for flags in (L.Q_STRICT_ORDER, 0):
            qa = AggQuery(one, calls, 60 * SEC, T0, tmax, flags=flags).run()
            qb = AggQuery(three, calls, 60 * SEC, T0, tmax, flags=flags).run()
            da, db = qa.dense_host(), qb.dense_host()
            for k in range(len(calls)):
                assert np.array_equal(da["cols"][k]["valid"], db["cols"][k]["valid"]), (calls, flags)
                assert np.array_equal(da["cols"][k]["values"].view(np.uint64), db["cols"][k]["values"].view(np.uint64)), (calls, flags)
            sa, sb = qa.stats()["path"], qb.stats()["path"]
            assert sa == sb, (calls, flags, sa, sb)
            if flags == 0 and calls == [("sum", 0), ("count", 0), ("max", 0)]:
                assert sb == 3
            qa.close(); qb.close()
    three.close(); one.close()


def test_overlapping_ordered_files_are_refused():
    t = T0 + np.arange(100, dtype=np.int64) * SEC
    f1 = {1: _series(t, {"v": (L.TYPE_FLOAT, np.arange(100.0), np.ones(100, bool))})}
    f2 = {1: _series(t[50:] + 1, {"v": (L.TYPE_FLOAT, np.arange(50.0), np.ones(50, bool))})}
    with pytest.raises(L.OgpuError) as ei:
        _open([(f1, False), (f2, False)])
    assert ei.value.status == L.OG_E_UNSUPPORTED and "overlap" in str(ei.value) and "sid 1" in str(ei.value)
    f3 = {1: _series(t, {"v": (L.TYPE_INT, np.arange(100), np.ones(100, bool))})}
    with pytest.raises(L.OgpuError) as ei:
        _open([(f1, False), (f3, True)])
    assert ei.value.status == L.OG_E_TYPE and '"v"' in str(ei.value)


# ---------------------------------------------------------------- 3. merged rows, bit for bit
@pytest.mark.parametrize("seed", [1, 2])
def test_merged_rows_equal_the_model(seed):
    files = _random_files(seed)
    sh = _open(files)
    _check_rows(sh, _model(files))
    sh.close()


def test_nan_and_infinities_in_out_of_order_rows():
    n = 3000
    t = T0 + np.arange(n, dtype=np.int64) * SEC
    v = np.linspace(1, 2, n)
    v[2500] = -np.inf                              # older file: -Inf only (a Gorilla page the encoder accepts)
    ordered = {7: _series(t, {"v": (L.TYPE_FLOAT, v, np.ones(n, bool))})}
    t2 = t[100:2900:7] + SEC // 3
    w = np.linspace(5, 6, t2.size)
    w[3] = np.nan                                  # NaN: the oracle encoder's Snappy route, transcoded at open
    w[(2600 - 100) // 7] = np.inf                  # lands in the merged segment that holds the -Inf row
    ooo = {7: _series(t2, {"v": (L.TYPE_FLOAT, w, np.ones(t2.size, bool))})}
    files = [(ordered, False), (ooo, True)]
    sh = _open(files)                               # +Inf and -Inf in one merged segment: raw page, not a refusal
    _check_rows(sh, _model(files))
    q = AggQuery(sh, [("count", 0)], 0, T0, T0 + n * SEC, flags=L.Q_STRICT_ORDER).run()
    assert q.dense_host()["cols"][0]["values"][0] == n + t2.size
    q.close(); sh.close()


def test_a_file_goes_through_og_tssp_parse():
    files = _random_files(3, n_series=4, rows=1800)
    ordered, _ = files[0]
    chunks = []
    for sid in sorted(ordered):
        s = ordered[sid]
        pages = {n: [] for n in s["cols"]}; tp, tmin, tmax = [], [], []
        for a in range(0, s["times"].size, 1000):
            b = min(a + 1000, s["times"].size)
            for n, (ty, v, ok) in s["cols"].items():
                pages[n].append(bytes(oracle.field_page_encode(ty, np.ascontiguousarray(v[a:b]), np.asarray(ok[a:b], np.uint8))))
            tp.append(bytes(oracle.time_page_encode(s["times"][a:b]))); tmin.append(int(s["times"][a])); tmax.append(int(s["times"][b - 1]))
        chunks.append(dict(sid=sid, tmin=tmin, tmax=tmax, columns=[(n.encode(), s["cols"][n][0], pages[n]) for n in sorted(s["cols"])], time=tp))
    image, _dir = tssp_file.build(chunks)
    sh = Shard.open_files([(image, False), (_file_desc(files[1][0]), True), (_file_desc(files[2][0]), True)])
    _check_rows(sh, _model(files))
    sh.close()


# ---------------------------------------------------------------- 4. aggregates against the restated file-set read
def test_aggregates_on_a_merged_shard():
    files = _random_files(4)
    model = _model(files)
    sh = _open(files)
    ex = sh.export()
    names = sorted({n for s in model.values() for n in s["cols"]})
    fv, iv_, bv = names.index("fv"), names.index("iv"), names.index("bv")
    tmin = min(int(s["times"][0]) for s in model.values())
    tmax = max(int(s["times"][-1]) for s in model.values())
    shapes = [[(f, fv)] for f in ALL6] + [[(f, iv_)] for f in ALL6] + [[(f, bv)] for f in ("count", "min", "max", "first", "last")]
    shapes += [[(f, fv) for f in ALL6], [("sum", iv_), ("count", bv), ("max", fv), ("first", iv_)]]
    for calls in shapes:
        for iv, off in ((60 * SEC, 0), (37 * SEC, 11 * SEC), (0, 0)):
            _compare(sh, files, calls, iv, tmin, tmax, offset=off, flags=L.Q_STRICT_ORDER)
        _compare(sh, files, calls, 60 * SEC, tmin, tmax, flags=0)
        _compare(sh, files, calls, 60 * SEC, tmin, tmax, group="series")  # untouched series: float sums bitwise
        _compare(sh, files, calls, 60 * SEC, tmin, tmax, ascending=False, flags=L.Q_STRICT_ORDER)
    # a query range that cuts a span, tag groups
    groups = np.arange(ex["sids"].size, dtype=np.uint32) % 3
    for calls in ([(f, fv) for f in ALL6], [("sum", iv_), ("min", iv_), ("last", bv)]):
        _compare(sh, files, calls, 45 * SEC, T0 + 333 * SEC, T0 + 1777 * SEC, flags=L.Q_STRICT_ORDER)
        _compare(sh, files, calls, 45 * SEC, tmin, tmax, group="map", series_group=groups, n_groups=3)
    sh.close()


def test_an_ordered_file_after_an_out_of_order_file_is_older():
    """files[] in file-sequence order may put an ordered file after an out-of-order one; the out-of-order file is still newer."""
    rng = np.random.default_rng(12)
    ta = T0 + np.arange(1500, dtype=np.int64) * SEC
    tc = T0 + np.arange(1500, 3000, dtype=np.int64) * SEC
    a = {s: _series(ta, {"v": (L.TYPE_FLOAT, rng.normal(0, 1, ta.size), np.ones(ta.size, bool)),
                         "i": (L.TYPE_INT, rng.integers(0, 99, ta.size), rng.random(ta.size) > 0.1)}) for s in (1, 2, 3)}
    c = {s: _series(tc, {"v": (L.TYPE_FLOAT, rng.normal(0, 1, tc.size), np.ones(tc.size, bool)),
                         "i": (L.TYPE_INT, rng.integers(0, 99, tc.size), rng.random(tc.size) > 0.1)}) for s in (1, 2, 3)}
    tb = np.unique(np.concatenate([ta[1200::3], tc[:400:2]]))  # shares times with both ordered files
    b = {s: _series(tb, {"v": (L.TYPE_FLOAT, rng.normal(100, 1, tb.size), rng.random(tb.size) > 0.2)}) for s in (1, 3)}
    files = [(a, False), (b, True), (c, False)]
    sh = _open(files)
    _check_rows(sh, _model(files))
    for calls in ([(f, 0) for f in ALL6], [("sum", 1), ("max", 1), ("count", 0)]):
        _compare(sh, files, calls, 60 * SEC, T0, T0 + 3000 * SEC, group="series", flags=L.Q_STRICT_ORDER)
    sh.close()


# ---------------------------------------------------------------- 5. WHERE
def test_where_without_shared_times_and_the_documented_deviation():
    rng = np.random.default_rng(9)
    n = 2000
    t = T0 + np.arange(n, dtype=np.int64) * SEC
    ordered = {s: _series(t, {"v": (L.TYPE_FLOAT, rng.normal(50, 30, n), np.ones(n, bool))}) for s in (1, 2, 3)}
    t2 = t[::5] + SEC // 2                          # no time shared with the ordered file
    ooo = {2: _series(t2, {"v": (L.TYPE_FLOAT, rng.normal(50, 30, t2.size), np.ones(t2.size, bool))})}
    files = [(ordered, False), (ooo, True)]
    sh = _open(files)
    for calls in ([("count", 0), ("sum", 0)], [("max", 0), ("first", 0)]):
        _compare(sh, files, calls, 60 * SEC, T0, T0 + n * SEC, where=[(0, ">", 40.0)], flags=L.Q_STRICT_ORDER)
        _compare(sh, files, calls, 60 * SEC, T0, T0 + n * SEC, where=[(0, ">", 40.0)], group="series")
    sh.close()
    # the newer row fails the filter, the older row with the same time passes it: the merged row (newer value) is filtered out.
    # The reference filters each file before merging and keeps the older row (DESIGN.md "Deviations").
    old = {1: _series(t[:10], {"v": (L.TYPE_FLOAT, np.full(10, 100.0), np.ones(10, bool))})}
    new = {1: _series(t[4:5], {"v": (L.TYPE_FLOAT, np.array([10.0]), np.ones(1, bool))})}
    files = [(old, False), (new, True)]
    sh = _open(files)
    q = AggQuery(sh, [("count", 0), ("min", 0)], 0, T0, T0 + 10 * SEC, filter=[("term", 0, ">", 50.0)], flags=L.Q_STRICT_ORDER).run()
    d = q.dense_host()
    assert d["cols"][0]["values"][0] == 9 and d["cols"][1]["values"][0] == 100.0
    ref, _ = oracle_files.scan_aggregate_files(files, q, [("v", ">", 50.0)])
    assert ref["cols"][0]["values"][0] == 10  # the reference's per-file filter keeps the older row
    q.close(); sh.close()


# ---------------------------------------------------------------- 6. merge_info
def test_merge_info_counts_equal_the_model():
    files = _random_files(6)
    model = _model(files)
    sh = _open(files)
    mi = sh.merge_info()
    ooo_rows = sum(s["times"].size for f, ooo in files if ooo for s in f.values())
    in_rows = sum(s["times"].size for f, _ in files for s in f.values())
    out_rows = sum(s["times"].size for s in model.values())
    merged_sids = {sid for f, ooo in files if ooo for sid in f}
    assert mi["n_files"] == 3 and mi["n_out_of_order_files"] == 2
    assert mi["series_merged"] == len(merged_sids)
    assert mi["out_of_order_rows"] == ooo_rows
    assert mi["rows_replaced"] == in_rows - out_rows
    assert mi["rows_after_merge"] == out_rows == sh.info()["n_rows"]
    ex = sh.export()
    assert mi["segments_kept"] + mi["segments_rewritten_out"] == ex["seg_tmin"].size
    assert mi["segments_rewritten_out"] > 0 and mi["segments_rewritten_in"] > 0 and mi["merge_ms"] > 0
    sh.close()


# ---------------------------------------------------------------- 7. batching
def test_batched_merge_gives_the_same_shard(monkeypatch):
    files = _random_files(7, n_series=20)
    one = _open(files)
    monkeypatch.setenv("OGPU_MERGE_BATCH_ROWS", "1500")
    many = _open(files)
    monkeypatch.delenv("OGPU_MERGE_BATCH_ROWS")
    ea, eb = one.export(), many.export()
    # the same pages in the same order; the batched build lays the new pages out batch by batch, so compare page bytes
    for k in ("sids", "series_seg_begin", "seg_tmin", "seg_tmax", "page_len", "col_types"):
        assert np.array_equal(ea[k], eb[k]), k
    for c in range(ea["page_off"].shape[0]):
        for g in range(ea["seg_tmin"].size):
            la = int(ea["page_len"][c][g])
            oa, ob = int(ea["page_off"][c][g]), int(eb["page_off"][c][g])
            assert np.array_equal(ea["data"][oa:oa + la], eb["data"][ob:ob + la]), (c, g)
    one.close(); many.close()


# ---------------------------------------------------------------- 8. refusals
def test_string_values_in_a_span_are_refused_and_kept_outside():
    n = 1200
    t = T0 + np.arange(n, dtype=np.int64) * SEC
    ok = np.ones(n, bool)
    ordered = {1: _series(t, {"s": (TYPE_STRING, None, ok), "v": (L.TYPE_FLOAT, np.arange(n, dtype=np.float64), ok)}),
               2: _series(t, {"s": (TYPE_STRING, None, ok), "v": (L.TYPE_FLOAT, np.arange(n, dtype=np.float64), ok)})}
    late = {1: _series(t[5:6] + 1, {"v": (L.TYPE_FLOAT, np.array([1.5]), np.ones(1, bool))})}
    with pytest.raises(L.OgpuError) as ei:
        _open([(ordered, False), (late, True)])
    assert ei.value.status == L.OG_E_UNSUPPORTED and '"s"' in str(ei.value)
    # an all-null string page inside a span holds no value to re-encode: accepted, the column stays null there
    nulls = {1: _series(t, {"s": (TYPE_STRING, None, np.zeros(n, bool)), "v": (L.TYPE_FLOAT, np.arange(n, dtype=np.float64), ok)})}
    sh = _open([(nulls, False), ({1: _series(t[5:6] + 1, {"v": (L.TYPE_FLOAT, np.array([1.5]), np.ones(1, bool))})}, True)])
    q = AggQuery(sh, [("count", 0), ("count", 1)], 0, T0, T0 + 2 * n * SEC, flags=L.Q_STRICT_ORDER).run()
    assert q.dense_host()["cols"][1]["values"].tolist() == [n + 1]
    q.close(); sh.close()
    # the late row in a series whose string pages lie outside every span: kept, count() still works
    late = {2: _series(t[-1:] + SEC, {"v": (L.TYPE_FLOAT, np.array([1.5]), np.ones(1, bool))})}
    sh = _open([(ordered, False), (late, True)])
    q = AggQuery(sh, [("count", 0), ("count", 1)], 0, T0, T0 + 2 * n * SEC, group="series", flags=L.Q_STRICT_ORDER).run()
    d = q.dense_host()
    assert d["cols"][0]["values"].tolist() == [n, n] and d["cols"][1]["values"].tolist() == [n, n + 1]
    q.close(); sh.close()


def test_a_time_repeated_inside_a_span_is_refused():
    t = T0 + np.arange(20, dtype=np.int64) * SEC
    ordered = {1: _series(t, {"v": (L.TYPE_FLOAT, np.arange(20.0), np.ones(20, bool))})}
    tl = np.array([t[3] + 1, t[3] + 1, t[4] + 1], np.int64)  # one file, one series, the same time twice
    late = {1: _series(tl, {"v": (L.TYPE_FLOAT, np.array([1.0, 2.0, 3.0]), np.ones(3, bool))})}
    with pytest.raises(L.OgpuError) as ei:
        _open([(ordered, False), (late, True)])
    assert ei.value.status == L.OG_E_CORRUPT and "twice" in str(ei.value)


# ---------------------------------------------------------------- 9. other entry points
def test_downsample_and_export_of_a_merged_shard():
    files = _random_files(8, with_bool=False)
    model = _model(files)
    sh = _open(files)
    ref = Shard.open_desc(_file_desc(model))
    names = sorted({n for s in model.values() for n in s["cols"]})
    fv = names.index("fv")
    tmin = min(int(s["times"][0]) for s in model.values())
    tmax = max(int(s["times"][-1]) for s in model.values())
    da, db = sh.downsample(fv, 60 * SEC, tmin, tmax), ref.downsample(fv, 60 * SEC, tmin, tmax)
    assert da.rows == db.rows > 0
    xa, xb = da.open(), db.open()
    for col in (1, 3, 4, 5):  # max, count, first, last of the window
        qa = AggQuery(xa, [("sum", col) if col == 3 else ("max", col)], 0, tmin - 60 * SEC, tmax, group="series", flags=L.Q_STRICT_ORDER).run()
        qb = AggQuery(xb, [("sum", col) if col == 3 else ("max", col)], 0, tmin - 60 * SEC, tmax, group="series", flags=L.Q_STRICT_ORDER).run()
        assert np.array_equal(qa.dense_host()["cols"][0]["values"], qb.dense_host()["cols"][0]["values"]), col
        qa.close(); qb.close()
    xa.close(); xb.close(); da.close(); db.close(); ref.close()
    # the merged shard's export reopens through og_shard_open and answers the same
    re = Shard.open_desc(oracle.shard_desc_from_export(sh.export()))
    for calls in ([(f, fv) for f in ALL6], [("sum", names.index("iv")), ("count", names.index("iv"))]):
        a = AggQuery(sh, calls, 60 * SEC, tmin, tmax, flags=L.Q_STRICT_ORDER).run()
        b = AggQuery(re, calls, 60 * SEC, tmin, tmax, flags=L.Q_STRICT_ORDER).run()
        ga, gb = a.dense_host(), b.dense_host()
        for k in range(len(calls)):
            assert np.array_equal(ga["cols"][k]["valid"], gb["cols"][k]["valid"])
            assert np.array_equal(ga["cols"][k]["values"].view(np.uint64), gb["cols"][k]["values"].view(np.uint64))
        a.close(); b.close()
    re.close(); sh.close()
