"""og_downsample_shard: every field of a shard under a per-type call list, in one call, checked against the CPU model in
downsample_model.py (the oracle's per-series aggregates, the union row rule, 1000-row segments, the oracle's encoders).

Every page is compared byte for byte with the model's, and decoded with the oracle to compare every cell and validity bit."""
import ctypes as C
import os
import struct
import subprocess

import numpy as np
import pytest

import downsample_model as M
import oracle
import time_grid as tg
from opengemini_b200 import _lib as L

T0, SEC = 1_700_000_000_000_000_000, 1_000_000_000
ALL6 = ["min", "max", "sum", "count", "first", "last"]
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(autouse=True)
def _device(request):
    if request.node.get_closest_marker("gpu"):  # the layout check at the end needs no device
        from opengemini_b200 import Shard
        Shard.init(0)


# ---------------------------------------------------------------- shards
def _string_page(valid, payload=b"\x10opaque-string-block-bytes"):
    """A string page as EncodeColumnHeader frames it: Full / Empty / bitmap header + an opaque block (never decoded)."""
    rows = len(valid)
    nil = int(rows - valid.sum())
    if nil == 0:
        return np.frombuffer(bytes([34]) + struct.pack(">I", rows) + payload, np.uint8)
    if nil == rows:
        return np.frombuffer(bytes([44]) + struct.pack(">I", rows), np.uint8)
    bm = np.packbits(valid.astype(np.uint8), bitorder="little").tobytes()
    return np.frombuffer(bytes([L.TYPE_STRING]) + struct.pack(">I", len(bm)) + bm + struct.pack(">II", 0, nil) + payload, np.uint8)


def _arr(p, n, dt):
    return np.ctypeslib.as_array(p, shape=(n,)).astype(dt) if n else np.empty(0, dt)


def _with_string_column(hs, seed):
    """The synthetic host shard plus a string field (named last in sort order) whose validity comes from `seed`.
    Returns (desc, [(times, valid)] per series)."""
    from opengemini_b200 import Shard
    d = hs.desc
    ng, nc, ns = d.n_segments, d.n_columns, d.n_series
    rng = np.random.default_rng(seed)
    data = [np.ctypeslib.as_array(d.data, shape=(d.data_len,)).copy()]
    pos = d.data_len
    po, pl, rows_of = [], [], [[] for _ in range(ns)]
    ssb = _arr(d.series_seg_begin, ns + 1, np.uint32)
    for s in range(ns):
        for g in range(ssb[s], ssb[s + 1]):
            t = oracle.time_page_decode(hs.page(nc, g))
            shape = (s + g) % 4
            valid = np.ones(t.size, bool) if shape == 0 else np.zeros(t.size, bool) if shape == 1 else rng.random(t.size) > 0.4
            page = _string_page(valid)
            data.append(page); po.append(pos); pl.append(page.size); pos += page.size
            rows_of[s].append((t, valid))
    cols = [(f"f{c}", int(d.columns[c].type), _arr(d.columns[c].page_off, ng, np.uint64), _arr(d.columns[c].page_len, ng, np.uint32))
            for c in range(nc)]
    cols.append((f"f{nc}", L.TYPE_STRING, po, pl))
    desc = Shard.desc(np.concatenate(data), _arr(d.sids, ns, np.uint64), ssb, _arr(d.seg_tmin, ng, np.int64), _arr(d.seg_tmax, ng, np.int64),
                      cols, _arr(d.time_page_off, ng, np.uint64), _arr(d.time_page_len, ng, np.uint32))
    return desc, [(np.concatenate([t for t, _ in r]), np.concatenate([v for _, v in r])) for r in rows_of]


def _rows_desc(series, names_types, seg_rows=1000):
    """A shard description from rows: series = [(times, {name: (values, valid)})], pages from the oracle's encoders."""
    from opengemini_b200 import Shard
    names = [n for n, _ in names_types]
    blob, pos = [], 0
    po = {n: [] for n in names}; pl = {n: [] for n in names}
    tpo, tpl, tmin, tmax, ssb = [], [], [], [], [0]

    def put(page):
        nonlocal pos
        blob.append(np.asarray(page, np.uint8)); off = pos; pos += len(page)
        return off, len(page)

    for t, cols in series:
        for a in range(0, t.size, seg_rows):
            b = min(t.size, a + seg_rows)
            for n, ty in names_types:
                v, ok = cols[n]
                o, ln = put(oracle.field_page_encode(ty, np.ascontiguousarray(v[a:b]), np.asarray(ok[a:b], np.uint8)))
                po[n].append(o); pl[n].append(ln)
            o, ln = put(oracle.time_page_encode(t[a:b]))
            tpo.append(o); tpl.append(ln); tmin.append(int(t[a])); tmax.append(int(t[b - 1]))
        ssb.append(len(tmin))
    return Shard.desc(np.concatenate(blob), np.arange(1, len(series) + 1), ssb, tmin, tmax,
                      [(n, ty, po[n], pl[n]) for n, ty in names_types], tpo, tpl)


# ---------------------------------------------------------------- model + comparison
def _model(desc, fields, ops, interval, tmin, tmax, strings=None):
    """fields: [(name, type)] of the shard; strings: {field index: [(times, valid)] per series}."""
    cols = M.schema(fields, ops)
    cells, grid = {}, None
    for fi, (_name, typ) in enumerate(fields):
        calls = ops.get(typ, [])
        if not calls:
            continue
        if typ == L.TYPE_STRING:
            continue
        grid, got = M.oracle_cells(desc, fi, calls, interval, tmin, tmax)
        for f in calls:
            cells[(fi, f)] = got[f]
    if strings:
        if grid is None:  # the string field's grid is the shard's: ask the oracle with any other field
            grid, _ = M.oracle_cells(desc, next(i for i, (_n, t) in enumerate(fields) if t != L.TYPE_STRING), ["count"], interval, tmin, tmax)
        for fi, rows in strings.items():
            if ops.get(L.TYPE_STRING):
                cells[(fi, "count")] = M.string_counts(rows, grid, tmin, tmax)
    return cols, M.expected(cols, cells, grid, desc.n_series) if cols else None


def _check(ds, cols, model):
    d = ds.desc
    got_cols, (tpo, tpl) = ds.columns()
    assert [(c[0], c[1]) for c in got_cols] == [(c[0], c[1]) for c in cols]
    if model is None:
        assert ds.rows == 0 and d.n_segments == 0
        return
    ng = d.n_segments
    assert ds.rows == model["rows"] and ng == len(model["seg_times"])
    assert list(_arr(d.series_seg_begin, d.n_series + 1, np.uint32)) == list(model["ssb"])
    data = ds.export()
    want_pages = M.pages(model)
    for g in range(ng):
        t = model["seg_times"][g]
        assert d.seg_tmin[g] == t[0] and d.seg_tmax[g] == t[-1], g
        page = data[tpo[g]:tpo[g] + tpl[g]]
        assert np.array_equal(oracle.time_page_decode(page), t), g
        assert page.tobytes() == want_pages[-1][g].tobytes(), ("time", g)
    for k, (name, typ, po, pl) in enumerate(got_cols):
        for g in range(ng):
            page = data[po[g]:po[g] + pl[g]]
            wv, wok = model["cols"][k][2][g]
            v, ok = oracle.field_page_decode(typ, page)
            assert np.array_equal(ok, wok), (name, g)
            want = M.cell_array(typ, wv)[wok]
            assert np.ascontiguousarray(v).tobytes() == np.ascontiguousarray(want).tobytes(), (name, g)  # bit-exact, float sums included
            assert page.tobytes() == want_pages[k][g].tobytes(), (name, g)


MIXED_OPS = {L.TYPE_FLOAT: ALL6, L.TYPE_INT: ["sum", "count", "max"], L.TYPE_BOOL: ["count", "first", "last"], L.TYPE_STRING: ["count"]}


# ---------------------------------------------------------------- cases
@pytest.mark.gpu
@pytest.mark.parametrize("interval", [5 * SEC, 60 * SEC])
def test_mixed_shard_matches_the_model(interval):
    from opengemini_b200 import Shard
    from opengemini_b200.downsample import downsample_shard
    cols = [(L.TYPE_FLOAT, L.SYNTH_F_HI, 0), (L.TYPE_FLOAT, L.SYNTH_F_LO, 150), (L.TYPE_INT, L.SYNTH_INT_WALK, 300), (L.TYPE_BOOL, L.SYNTH_BOOL, 500)]
    hs = oracle.HostShard(5, 3300, cols, t0=T0, dt=SEC, seed=41)
    desc, srows = _with_string_column(hs, 7)
    fields = [(f"f{c}", t) for c, (t, _d, _n) in enumerate(cols)] + [("f4", L.TYPE_STRING)]
    sh = Shard.open_desc(desc)
    tmin, tmax = T0 + 17 * SEC, T0 + 3211 * SEC
    want_cols, model = _model(desc, fields, MIXED_OPS, interval, tmin, tmax, strings={4: srows})
    ds = sh.downsample_shard(interval, tmin, tmax, MIXED_OPS)
    _check(ds, want_cols, model)
    assert [c[0] for c in want_cols][:3] == ["count_f0", "count_f1", "count_f2"]
    # the Python wrapper returns the same shard
    w = downsample_shard(sh, interval, tmin, tmax, MIXED_OPS)
    assert w["names"] == [c[0] for c in want_cols] and w["rows"] == ds.rows
    assert w["data"][:w["data_len"]].cpu().numpy().tobytes() == ds.export().tobytes()
    assert list(w["series_seg_begin"]) == list(model["ssb"])
    ds.close(); sh.close()


@pytest.mark.gpu
@pytest.mark.parametrize("interval", [SEC, 3 * SEC])
def test_fields_in_disjoint_windows_give_null_cells(interval):
    """Two fields valid in alternating 37-row blocks and a third block where neither is: rows carry null cells in one column or
    the other, segments (several per series at 1 s) start and end on either, and windows with no value at all are dropped."""
    from opengemini_b200 import Shard
    rng = np.random.default_rng(5)
    series = []
    for s in range(3):
        n = 3100 + 211 * s
        t = T0 + np.arange(n, dtype=np.int64) * SEC
        blk = (np.arange(n) + 13 * s) // 37 % 3
        series.append((t, {"a": (rng.normal(50, 9, n), blk == 0), "b": (rng.integers(-99, 99, n).cumsum(), blk == 1)}))
    nt = [("a", L.TYPE_FLOAT), ("b", L.TYPE_INT)]
    desc = _rows_desc(series, nt)
    sh = Shard.open_desc(desc)
    ops = {L.TYPE_FLOAT: ["max", "count", "first"], L.TYPE_INT: ["min", "sum", "last"]}
    tmin, tmax = T0, T0 + 4000 * SEC
    want_cols, model = _model(desc, nt, ops, interval, tmin, tmax)
    ds = sh.downsample_shard(interval, tmin, tmax, ops)
    _check(ds, want_cols, model)
    nulls = [sum(int((~ok).sum()) for _v, ok in segs) for _n, _t, segs in model["cols"]]
    assert min(nulls) > 0  # every column has null cells
    if interval == SEC:
        assert model["ssb"][1] >= 2
    ds.close(); sh.close()


@pytest.mark.gpu
def test_column_subsets_empty_lists_and_all_null_fields():
    from opengemini_b200 import Shard
    cols = [(L.TYPE_FLOAT, L.SYNTH_F_HI, 0), (L.TYPE_INT, L.SYNTH_INT_WALK, 1000), (L.TYPE_BOOL, L.SYNTH_BOOL, 100), (L.TYPE_FLOAT, L.SYNTH_F_LO, 1000)]
    hs = oracle.HostShard(4, 2500, cols, t0=T0, dt=SEC, seed=23)
    sh = Shard.open_desc(hs.desc, keepalive=hs)
    fields = [(f"f{c}", t) for c, (t, _d, _n) in enumerate(cols)]
    tmin, tmax = T0 + 100 * SEC, T0 + 2400 * SEC
    cases = [
        {L.TYPE_FLOAT: ["sum", "last"]},                         # int and bool have no entry: dropped; f3 all null
        {L.TYPE_FLOAT: ["min"], L.TYPE_INT: [], L.TYPE_BOOL: ["max", "min"]},  # an empty list drops int
        {L.TYPE_INT: ["count", "sum"]},                          # the only field is all null: columns, no rows
        {L.TYPE_STRING: ["count"]},                               # no field of the type: no columns at all
        {},
    ]
    for ops in cases:
        want_cols, model = _model(hs.desc, fields, ops, 10 * SEC, tmin, tmax)
        ds = sh.downsample_shard(10 * SEC, tmin, tmax, ops)
        _check(ds, want_cols, model)
        if ops.get(L.TYPE_INT) == ["count", "sum"]:
            assert ds.desc.n_columns == 2 and ds.rows == 0 and ds.desc.n_segments == 0
        ds.close()
    sh.close()


@pytest.mark.gpu
@pytest.mark.parametrize("interval", [SEC, 2 * SEC, 3 * SEC, 7 * SEC])
def test_segment_cuts_and_ranges_cut_mid_segment(interval):
    """More than 1000 kept windows per series (several output segments), a range that starts and ends inside source segments,
    and intervals that do (1 s, 2 s) and do not (3 s, 7 s) divide the 1000 s a source segment spans."""
    from opengemini_b200 import Shard
    cols = [(L.TYPE_FLOAT, L.SYNTH_F_HI, 20), (L.TYPE_INT, L.SYNTH_INT_WALK, 0)]
    hs = oracle.HostShard(3, 7500, cols, t0=T0, dt=SEC, seed=61)
    sh = Shard.open_desc(hs.desc, keepalive=hs)
    fields = [("f0", L.TYPE_FLOAT), ("f1", L.TYPE_INT)]
    ops = {L.TYPE_FLOAT: ALL6, L.TYPE_INT: ALL6}
    tmin, tmax = T0 + 1234 * SEC, T0 + 6789 * SEC
    want_cols, model = _model(hs.desc, fields, ops, interval, tmin, tmax)
    ds = sh.downsample_shard(interval, tmin, tmax, ops)
    _check(ds, want_cols, model)
    if interval <= 3 * SEC:
        assert model["ssb"][1] >= 2
    ds.close(); sh.close()


@pytest.mark.gpu
@pytest.mark.parametrize("typ,dist,nulls", [(L.TYPE_FLOAT, L.SYNTH_F_HI, 0), (L.TYPE_INT, L.SYNTH_INT_WALK, 0), (L.TYPE_FLOAT, L.SYNTH_F_HI, 400)],
                         ids=["float", "int", "float_nulls"])
def test_agrees_with_og_downsample(typ, dist, nulls):
    """The two entry points differ only in column names and order, with nulls too (3-second windows whose rows are all null)."""
    from opengemini_b200 import Shard
    sh = Shard.synth(5, 4321, [(typ, dist, nulls)], t0=T0, dt=SEC, seed=13)
    tmin, tmax, ivl = T0 + 5 * SEC, T0 + 4310 * SEC, 3 * SEC
    a = sh.downsample(0, ivl, tmin, tmax)
    b = sh.downsample_shard(ivl, tmin, tmax, {typ: ALL6})
    ca, ta = a.columns()
    cb, tb = b.columns()
    assert sorted(c[0] for c in ca) == [c[0] for c in cb]
    assert a.rows == b.rows and a.desc.n_segments == b.desc.n_segments
    ng = a.desc.n_segments
    assert list(_arr(a.desc.series_seg_begin, 6, np.uint32)) == list(_arr(b.desc.series_seg_begin, 6, np.uint32))
    assert [a.desc.seg_tmin[g] for g in range(ng)] == [b.desc.seg_tmin[g] for g in range(ng)]
    assert [a.desc.seg_tmax[g] for g in range(ng)] == [b.desc.seg_tmax[g] for g in range(ng)]
    da, db = a.export(), b.export()
    byname = {c[0]: c for c in cb}
    for name, ctyp, po, pl in ca + [("time", L.TYPE_INT, *ta)]:
        qpo, qpl = (tb if name == "time" else byname[name][2:])
        if name != "time":
            assert byname[name][1] == ctyp
        for g in range(ng):
            assert da[po[g]:po[g] + pl[g]].tobytes() == db[qpo[g]:qpo[g] + qpl[g]].tobytes(), (name, g)
    a.close(); b.close(); sh.close()


@pytest.mark.gpu
def test_round_trip_coarser_queries():
    """Reopened in place, the output answers coarser queries like the source: sum(count_x) == count(x), max(max_x) == max(x),
    first(first_x) == first(x) with the fine window start of first(x)'s row as its time."""
    from opengemini_b200 import AggQuery, Shard
    cols = [(L.TYPE_FLOAT, L.SYNTH_F_HI, 100), (L.TYPE_INT, L.SYNTH_INT_WALK, 250)]
    sh = Shard.synth(4, 6000, cols, t0=T0, dt=SEC, seed=77)
    fine, coarse = 5 * SEC, 60 * SEC
    tmin = (T0 // coarse + 1) * coarse
    tmax = tmin + 90 * coarse - 1
    ds = sh.downsample_shard(fine, tmin, tmax, {L.TYPE_FLOAT: ALL6, L.TYPE_INT: ALL6})
    names = [c[0] for c in ds.columns()[0]]
    x = ds.open()
    for f in (0, 1):
        q1 = AggQuery(x, [("sum", names.index(f"count_f{f}")), ("max", names.index(f"max_f{f}")), ("first", names.index(f"first_f{f}"))],
                      coarse, tmin, tmax, group="series", flags=L.Q_QUERY_GRID).run().dense_host()
        # (one grid over the query range: the output's last row is a window start, the source's a later time)
        q0 = AggQuery(sh, [("count", f), ("max", f), ("first", f)], coarse, tmin, tmax, group="series", flags=L.Q_QUERY_GRID).run().dense_host()
        assert q1["n_buckets"] == q0["n_buckets"] and q1["start"] == q0["start"]
        for k in range(3):
            assert np.array_equal(q1["cols"][k]["valid"], q0["cols"][k]["valid"]), (f, k)
            m = q0["cols"][k]["valid"].astype(bool)
            assert np.array_equal(q1["cols"][k]["values"].view(np.uint64)[m], q0["cols"][k]["values"].view(np.uint64)[m]), (f, k)
        m = q0["cols"][2]["valid"].astype(bool)
        t0 = q0["cols"][2]["times"][m]
        assert np.array_equal(q1["cols"][2]["times"][m], t0 - (t0 % fine)), f
    x.close(); ds.close(); sh.close()


@pytest.mark.gpu
def test_merged_input():
    """A shard opened from an ordered and an out-of-order file: the result is the model's over the merged rows (the merged
    shard's export, whose correctness the merge tests establish)."""
    from opengemini_b200 import Shard
    rng = np.random.default_rng(19)
    ordered, late = [], []
    for s in range(4):
        n = 2600
        t = T0 + np.arange(n, dtype=np.int64) * SEC
        ordered.append((t, {"fv": (rng.normal(100, 20, n), rng.random(n) > 0.05), "iv": (rng.integers(-500, 500, n).cumsum(), rng.random(n) > 0.1)}))
        k = 300
        t2 = np.unique(T0 + rng.integers(-100, n + 100, k) * SEC + np.where(rng.random(k) < 0.3, SEC // 2, 0))
        late.append((t2, {"fv": (rng.normal(0, 5, t2.size), rng.random(t2.size) > 0.3), "iv": (rng.integers(-9, 9, t2.size), rng.random(t2.size) > 0.3)}))
    nt = [("fv", L.TYPE_FLOAT), ("iv", L.TYPE_INT)]
    sh = Shard.open_files([(_rows_desc(ordered, nt), False), (_rows_desc(late, nt), True)])
    assert sh.merge_info()["out_of_order_rows"] > 0
    merged = oracle.shard_desc_from_export(sh.export())
    ops = {L.TYPE_FLOAT: ALL6, L.TYPE_INT: ["count", "sum", "first"]}
    tmin, tmax, ivl = T0 - 200 * SEC, T0 + 2800 * SEC, 2 * SEC
    want_cols, model = _model(merged, nt, ops, ivl, tmin, tmax)  # the export's columns are fv, iv in that order
    ds = sh.downsample_shard(ivl, tmin, tmax, ops)
    _check(ds, want_cols, model)
    ds.close(); sh.close()


@pytest.mark.gpu
def test_refusals():
    from opengemini_b200 import AggQuery, Shard
    sh = Shard.synth(2, 500, [(L.TYPE_FLOAT, L.SYNTH_F_HI, 0), (L.TYPE_BOOL, L.SYNTH_BOOL, 0)], t0=T0, dt=SEC, seed=3)
    tmin, tmax = T0, T0 + 499 * SEC

    def status(ops, interval=10 * SEC, lo=tmin, hi=tmax):
        with pytest.raises(L.OgpuError) as e:
            sh.downsample_shard(interval, lo, hi, ops)
        return e.value.status, str(e.value)

    st, msg = status({L.TYPE_STRING: ["count", "first"]})
    assert st == L.OG_E_UNSUPPORTED and "string" in msg and "count" in msg
    assert status({L.TYPE_BOOL: ["count", "sum"]})[0] == L.OG_E_INVAL
    assert status({L.TYPE_FLOAT: [99]})[0] == L.OG_E_INVAL
    assert status({L.TYPE_FLOAT: ["min", "min"]})[0] == L.OG_E_INVAL
    assert status({L.TYPE_FLOAT: ["min"]}, interval=0)[0] == L.OG_E_INVAL
    # a type listed twice (not expressible through a dict): build the descriptor by hand
    f = (C.c_int32 * 1)(L.AGG_MIN)
    arr = (L.DownsampleOps * 2)((L.TYPE_FLOAT, 1, C.cast(f, L.i32p)), (L.TYPE_FLOAT, 1, C.cast(f, L.i32p)))
    h = C.c_void_p()
    assert L.lib().og_downsample_shard(sh.h, C.byref(L.DownsampleDesc(10 * SEC, tmin, tmax, 2, arr)), C.byref(h)) == L.OG_E_INVAL
    assert not h.value
    sh.close()
    # a range whose last window is clamped at MAX_TIME: the refusal og_query_create gives
    t0 = tg.MAX_TIME - 7 * 299
    series = [(t0 + np.arange(300, dtype=np.int64) * 7, {"v": (np.arange(300, dtype=np.float64), np.ones(300, bool))})]
    ch = Shard.open_desc(_rows_desc(series, [("v", L.TYPE_FLOAT)]))
    lo, hi = tg.MIN_TIME, tg.MAX_TIME
    with pytest.raises(L.OgpuError) as e0:
        AggQuery(ch, [("count", 0)], 100, lo, hi, group="series")
    with pytest.raises(L.OgpuError) as e1:
        ch.downsample_shard(100, lo, hi, {L.TYPE_FLOAT: ["count"]})
    assert e1.value.status == e0.value.status == L.OG_E_UNSUPPORTED
    assert str(e1.value).split(") ", 1)[1] == str(e0.value).split(") ", 1)[1]  # same detail message
    ch.close()


def test_struct_layouts_match_the_header(tmp_path):
    """sizeof / offsetof of the new descriptor structs as the C compiler sees include/ogpu.h == the ctypes mirror."""
    pairs = {"og_downsample_ops": L.DownsampleOps, "og_downsample_desc": L.DownsampleDesc}
    lines = ["#include <stdio.h>", "#include <stddef.h>", f'#include "{os.path.join(ROOT, "include", "ogpu.h")}"', "int main(void) {"]
    for cname, cls in pairs.items():
        lines.append(f'  printf("{cname} %zu\\n", sizeof({cname}));')
        for fname, _t in cls._fields_:
            lines.append(f'  printf("{cname}.{fname} %zu\\n", offsetof({cname}, {fname}));')
    lines += ["  return 0;", "}"]
    src = tmp_path / "layout.c"
    src.write_text("\n".join(lines))
    exe = tmp_path / "layout"
    subprocess.run(["gcc", "-std=c11", "-o", str(exe), str(src)], check=True)
    out = subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout
    seen = dict(line.split() for line in out.strip().splitlines())
    for cname, cls in pairs.items():
        assert int(seen[cname]) == C.sizeof(cls), cname
        for fname, _t in cls._fields_:
            assert int(seen[f"{cname}.{fname}"]) == getattr(cls, fname).offset, f"{cname}.{fname}"
