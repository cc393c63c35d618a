"""Histories of one open shard: appends of ordered and out-of-order files, compactions at changing R, refusals, writes, downsamples
and queries in between, in the order a store runs them.

Each test is one scripted history aimed at one interaction between these mutations.  After every step _step_check holds the shard
to the same references: its rows against _model over every file so far (compaction does not change a file set's rows), og_shard_info
and, after an append or a re-cut, a data region of live pages only, the compaction model after a compaction, that call's counters in og_shard_merge_info after an
append, and every aggregate path against segment_shards.window_model (which does not depend on how rows are cut into segments) and,
in the reference's order, against the oracle over the shard's export."""
import os

import numpy as np
import pytest

import compact_model as cm
import oracle
import segment_shards as ss
from opengemini_b200 import AggQuery, Shard, write_tssp
from opengemini_b200 import _lib as L
from test_gpu_append import _cols, _data_excess, _descs, _flush, _late, _same_directory_and_pages, _snapshot, _unchanged
from test_gpu_device_memory import _NoLeak
from test_gpu_out_of_order import ALL6, SEC, T0, _check_rows, _file_desc, _model, _series

pytestmark = pytest.mark.gpu
IV = 60 * SEC


@pytest.fixture(scope="module", autouse=True)
def _device():
    Shard.init(0)


def _window_series(model, names, where=None):
    """the _model dict as the series list segment_shards.window_model takes: series in sid order, columns in name order.
    where = (name, op, const): a row counts only where that column is non-null and passes ("<" or ">")."""
    out = []
    for sid in sorted(model):
        s = model[sid]
        keep = np.ones(s["times"].size, bool)
        if where:
            _ty, v, ok = s["cols"][where[0]]
            keep = ok & ((v > where[2]) if where[1] == ">" else (v < where[2]))
        out.append(dict(times=s["times"], cols=[(s["cols"][n][1], s["cols"][n][2] & keep) for n in names]))
    return out


def _step_check(sh, files, before=None):
    """The shard after one step of a history.  before: after a compaction dict(want=cm.expected(export before, R), info=its
    og_compact_info, merge_info=og_shard_merge_info before); after an append dict(step=that call's files, n_rows=n_rows before)."""
    model = _model(files)
    names = sorted({n for s in model.values() for n in s["cols"]})
    types = {n: t for s in model.values() for n, (t, _v, _k) in s["cols"].items()}
    _check_rows(sh, model)
    ex, info = sh.export(), sh.info()
    tmin = min(int(s["times"][0]) for s in model.values())
    tmax = max(int(s["times"][-1]) for s in model.values())
    assert info["n_series"] == len(model) and info["n_rows"] == sum(s["times"].size for s in model.values())
    assert (info["tmin"], info["tmax"]) == (tmin, tmax)
    assert info["n_segments"] == ex["seg_tmin"].size
    before = before or {}
    if "step" in before or before.get("info", {}).get("series_rewritten"):
        assert _data_excess(sh) == 0  # live pages only; an open keeps the files' bytes as they were copied in
    if "want" in before:
        cm.assert_matches(ex, before["want"])
        assert {k: v for k, v in before["info"].items() if k != "compact_ms"} == before["want"]["info"]
        assert sh.merge_info() == before["merge_info"]
    if "step" in before:
        step, mi = before["step"], sh.merge_info()
        assert mi["n_files"] == len(step) and mi["n_out_of_order_files"] == sum(o for _, o in step)
        assert mi["out_of_order_rows"] == sum(s_["times"].size for f, o in step if o for s_ in f.values())
        assert mi["rows_after_merge"] == info["n_rows"]
        assert mi["series_merged"] == len({sid for f, o in step if o for sid in f})
        in_rows = before["n_rows"] + sum(s_["times"].size for f, _ in step for s_ in f.values())
        assert mi["rows_replaced"] == in_rows - mi["rows_after_merge"]
        assert mi["segments_kept"] + mi["segments_rewritten_out"] == ex["seg_tmin"].size
    # ---- what the layout makes eligible, from the directory and the page headers
    nc, ssb, ns = ex["col_types"].size, ex["series_seg_begin"].astype(np.int64), ex["sids"].size

    def page(c, g):
        o = int(ex["page_off"][c][g])
        return ex["data"][o:o + int(ex["page_len"][c][g])]

    tps = [page(nc, g) for g in range(ex["seg_tmin"].size)]
    one_row = [p[0] == 18 for p in tps]  # [18][t LE]: the time page of a one-row segment
    rows = [1 if o else int.from_bytes(p[1:5].tobytes(), "big") for p, o in zip(tps, one_row)]
    const_dt = [not o and p[5] >> 4 == 1 for p, o in zip(tps, one_row)]  # [32][u32 rows][0x10 ...]: a const-delta time page
    per = np.diff(ssb)
    regular = len(set(per.tolist())) == 1 and all(
        np.array_equal(ex[k][ssb[u]:ssb[u + 1]], ex[k][ssb[0]:ssb[1]]) for u in range(ns) for k in ("seg_tmin", "seg_tmax"))
    cols_ok = all(d or o for d, o in zip(const_dt, one_row)) and max(rows) <= 1024

    def il_ok(c):  # some segment k_fused_il takes: a Gorilla or raw float page without nulls over a const-delta time page
        def takes(p, g):
            return p.size >= 16 and p[0] == 31 and ((p[5] >> 4 == 3 and p[6] == 0x10) or (p[5] >> 4 == 0 and p.size == 6 + 8 * rows[g]))
        return any(ex["page_len"][c][g] and takes(page(c, g), g) and const_dt[g] and rows[g] >= 2 for g in range(len(tps)))

    desc = oracle.shard_desc_from_export(ex)
    sids = ex["sids"].astype(np.int64)
    groupings = {"all": np.zeros(ns, np.int64), "series": np.arange(ns), "map": sids % 3}
    models = {}

    def check(calls, path=None, where=None, group="all", **kw):
        g = groupings[group]
        if group == "map":
            kw.update(series_group=g.astype(np.uint32), n_groups=int(g.max()) + 1)
        flt = [("term", names.index(where[0]), where[1], where[2])] if where else None
        q = AggQuery(sh, calls, IV, tmin, tmax, filter=flt, group=group, **kw).run()
        got, st = q.dense_host(), q.stats()
        strict = bool(kw.get("flags", 0) & L.Q_STRICT_ORDER) or group != "all"
        ref = oracle.scan(desc, q.desc, threads=1) if strict else None
        q.close()
        label = f"{calls} {group} {kw.get('flags', 0)} {where} {kw.get('ascending', True)}"
        if path is not None:
            assert st["path"] == path, (label, st["path"])
        for k, (f, c) in enumerate(calls):
            key = (c, group, where)
            if key not in models:
                models[key] = ss.window_model(_window_series(model, names, where), c, types[names[c]], IV, 0, tmin, tmax, g)
            sub = dict(n_buckets=got["n_buckets"], start=got["start"], cols=[got["cols"][k]])
            ss.check_against_model(sub, [(f, c)], models[key], types[names[c]], label, multi=len(calls) > 1)
            if ref is not None:  # the reference's order: bit for bit, float sums included
                rv = ref["cols"][k]["valid"].astype(bool)
                assert np.array_equal(got["cols"][k]["valid"].astype(bool), rv), label
                assert np.array_equal(got["cols"][k]["values"].view(np.uint64)[rv], ref["cols"][k]["values"][rv]), (label, f)
                if got["cols"][k]["times"] is not None:
                    assert np.array_equal(got["cols"][k]["times"][rv], ref["cols"][k]["times"][rv]), (label, f)
        return st

    floats = [c for c, n in enumerate(names) if types[n] == L.TYPE_FLOAT]
    for f in floats:
        fc, all6 = [("sum", f), ("count", f), ("max", f)], [(x, f) for x in ALL6]
        ok = il_ok(f)
        # the first query of the column after a mutation: its interleaved copy is built for the layout the shard has now
        st = check(fc, path=(3 if regular else 2) if ok else 1)
        if ok:
            assert st["il_state"] == 1, names[f]
        check(all6, path=2 if ok else 1, flags=L.Q_STRICT_ORDER)
        check(fc, path=1, flags=L.Q_NO_FAST)
        check(fc, path=0, flags=L.Q_NO_FUSED | L.Q_STRICT_ORDER)
        check(all6, group="series")
        check(fc, group="map")
        check(all6, flags=L.Q_STRICT_ORDER, ascending=False)
    ints = [c for c, n in enumerate(names) if types[n] == L.TYPE_INT]
    for i in ints:
        check([("sum", i), ("min", i), ("last", i)], path=1, flags=L.Q_STRICT_ORDER)
        check([("sum", i), ("max", i)], group="map", ascending=False)
    if floats and ints:
        f0 = names[floats[0]]
        thr = float(np.median(np.concatenate([s["cols"][f0][1][s["cols"][f0][2]] for s in model.values()])))
        two = [("count", floats[0]), ("sum", ints[0])]
        check(two, path=5 if cols_ok else 4, where=(f0, ">", thr), flags=L.Q_STRICT_ORDER)
        os.environ["OGPU_NO_COLS"] = "1"
        try:
            check(two, path=4, where=(f0, ">", thr), flags=L.Q_STRICT_ORDER)
        finally:
            del os.environ["OGPU_NO_COLS"]
    return model


def _compact(sh, files, R):
    """one compaction step: the model of the export before it, the call, _step_check"""
    b = dict(want=cm.expected(sh.export(), R), merge_info=sh.merge_info())
    b["info"] = sh.compact(R)
    _step_check(sh, files, b)
    return b["info"]


def _append(sh, files, step):
    """one append step: the call, the files joining the model, _step_check"""
    b = dict(step=step, n_rows=sh.info()["n_rows"])
    sh.append_files(_descs(step))
    files += step
    _step_check(sh, files, b)


def _refused(call, status, text, sh, files):
    snap = _snapshot(sh)
    with pytest.raises(L.OgpuError) as ei:
        call()
    assert ei.value.status == status, str(ei.value)
    assert text in str(ei.value), str(ei.value)
    _unchanged(sh, snap)
    _step_check(sh, files)


def _after_last(rng, model, sids, n, gap=SEC, present=("fv", "iv")):
    """an ordered flush of n rows per series, 1 s apart, the first `gap` after the series' last time"""
    return {sid: _series(int(model[sid]["times"][-1]) + gap + SEC * np.arange(n, dtype=np.int64), _cols(rng, n, present, 0.0))
            for sid in sids}


# ---------------------------------------------------------------- 1
def test_compact_then_flush_then_compact():
    """The flush rule's last time of a series after a re-cut: a flush 1 ns after it is taken, one at it is refused naming the sid
    and leaves the shard as it was; the next compaction re-cuts only the tails, and a non-last segment of R - 1 rows is re-cut."""
    rng = np.random.default_rng(101)
    sids = [3, 7, 11, 19]
    files = [(_flush(rng, sids, 0, 2500, ("fv", "iv"), 0.0), False), (_flush(rng, sids, 2500, 40, ("fv", "iv"), 0.0), False),
             (_flush(rng, sids, 2540, 25, ("fv", "iv"), 0.0), False)]
    sh = Shard.open_files(_descs(files))
    _step_check(sh, files)
    assert _compact(sh, files, 1000)["series_rewritten"] == len(sids)          # [1000, 1000, 565]
    model = _model(files)
    bad = _after_last(rng, model, sids, 30)
    bad[7] = _series(model[7]["times"][-1] + SEC * np.arange(30, dtype=np.int64), _cols(rng, 30, ("fv", "iv"), 0.0))
    _refused(lambda: sh.append_files(_descs([(bad, False)])), L.OG_E_UNSUPPORTED, "sid 7", sh, files)
    ok = _after_last(rng, model, sids, 30)
    ok[3] = _series(model[3]["times"][-1] + 1 + SEC * np.arange(30, dtype=np.int64), _cols(rng, 30, ("fv", "iv"), 0.0))
    _append(sh, files, [(ok, False)])
    info = _compact(sh, files, 1000)                                             # only the tails: [565, 30] -> [595]
    assert info["series_rewritten"] == len(sids) and info["segments_kept"] == 2 * len(sids) and info["rows_rewritten"] == 595 * len(sids)
    _append(sh, files, [(_after_last(rng, _model(files), sids, 404), False)])   # [1000, 1000, 595, 404]
    assert _compact(sh, files, 1000)["segments_kept"] == 2 * len(sids)          # [1000, 1000, 999]
    _append(sh, files, [(_after_last(rng, _model(files), sids, 30), False)])    # a non-last segment of R - 1 rows
    info = _compact(sh, files, 1000)
    assert info["segments_rewritten_in"] == 2 * len(sids) and info["segments_rewritten_out"] == 2 * len(sids)
    assert sh.compact(1000)["series_rewritten"] == 0
    sh.close()


# ---------------------------------------------------------------- 2
def test_out_of_order_rows_into_compacted_short_segments():
    """Out-of-order spans that land on 7-row compacted segments, on half-second times and across a series' last time: that
    series' last time moves past its last ordered row, so an ordered flush starting between the two is refused and one after the
    late rows is taken; then compactions at R = 7 (with a non-last segment of R - 1 rows), 1000 and 1."""
    rng = np.random.default_rng(102)
    sids = [1, 2, 3, 4]
    files = [(_flush(rng, sids, 0, 203, ("fv", "iv"), 0.0), False)]
    sh = Shard.open_files(_descs(files))
    _step_check(sh, files)
    _compact(sh, files, 7)                                                       # 29 segments of 7 rows per series
    t = T0 + (np.array([50.5, 51.5, 52.5, 120, 202.5, 203.5, 206]) * SEC).astype(np.int64)
    late = {2: _series(t, _cols(rng, t.size, ("fv", "iv"), 0.2))}
    _append(sh, files, [(late, True)])
    model = _model(files)
    assert model[2]["times"][-1] == T0 + 206 * SEC
    between = {2: _series(T0 + 204 * SEC + SEC * np.arange(5, dtype=np.int64), _cols(rng, 5, ("fv", "iv"), 0.0))}
    _refused(lambda: sh.append_files(_descs([(between, False)])), L.OG_E_UNSUPPORTED, "sid 2", sh, files)
    _append(sh, files, [(_after_last(rng, model, sids, 14), False)])            # sid 1: 217 rows, a multiple of 7
    _compact(sh, files, 7)
    _append(sh, files, [(_after_last(rng, _model(files), [1, 3], 6), False)])   # [7, ..., 7, 6]
    _append(sh, files, [(_after_last(rng, _model(files), [1, 3], 5), False)])   # [7, ..., 7, 6, 5]
    info = _compact(sh, files, 7)
    assert info["segments_kept"] >= 31                                           # sid 1 keeps its 31 full segments
    _compact(sh, files, 1000)
    info = _compact(sh, files, 1)
    assert info["series_rewritten"] == len(sids) and sh.info()["n_segments"] == sh.info()["n_rows"]
    sh.close()


# ---------------------------------------------------------------- 3
def test_interleaved_copies_across_every_mutation():
    """Interleaved copies of two float columns, built before every mutation: an append, a compaction, a compaction refused for a
    live query, an append refused by the flush rule (the answer after it is the one before it, bit for bit); every first query
    after a mutation rebuilds the copy for the new layout, and the folded path is back once the shard is compact."""
    rng = np.random.default_rng(103)
    sids = list(range(40, 56))

    def flush(t_lo, n):
        f = _flush(rng, sids, t_lo, n, ("fv", "iv"), 0.0)
        for s_ in f.values():
            s_["cols"]["gv"] = (L.TYPE_FLOAT, np.round(rng.normal(0, 50, n), 2) + rng.random(n) * 1e-7, np.ones(n, bool))
        return f

    files = [(flush(0, 2000), False)]
    sh = Shard.open_files(_descs(files))
    _step_check(sh, files)                        # builds both copies: folded and strict order
    _append(sh, files, [(flush(2000, 300), False)])
    _append(sh, files, [(flush(2300, 300), False)])
    _compact(sh, files, 1000)                     # [1000, 1000, 600]
    _append(sh, files, [(flush(2600, 300), False)])
    q = AggQuery(sh, [("count", 0)], 0, T0, T0 + 9000 * SEC)
    _refused(lambda: sh.compact(), L.OG_E_STATE, "queries", sh, files)
    q.close()
    _compact(sh, files, 1000)                     # [1000, 1000, 900]
    folded = AggQuery(sh, [("sum", 0), ("count", 0), ("max", 0)], IV, T0, T0 + 2899 * SEC).run()
    d0 = [c["values"].view(np.uint64).copy() for c in folded.dense_host()["cols"]]
    assert folded.stats()["path"] == 3
    folded.close()
    _refused(lambda: sh.append_files(_descs([(flush(2899, 10), False)])), L.OG_E_UNSUPPORTED, "sid 40", sh, files)
    again = AggQuery(sh, [("sum", 0), ("count", 0), ("max", 0)], IV, T0, T0 + 2899 * SEC).run()
    assert all(np.array_equal(c["values"].view(np.uint64), x) for c, x in zip(again.dense_host()["cols"], d0))
    assert again.stats()["path"] == 3 and again.stats()["il_state"] == 1
    again.close()
    _append(sh, files, [(flush(2900, 150), False)])
    _append(sh, files, [(flush(3050, 150), False)])
    _compact(sh, files, 1000)                     # [1000, 1000, 1000, 200]
    q = AggQuery(sh, [("sum", 0), ("count", 0), ("max", 0)], IV, T0, T0 + 3199 * SEC).run()
    assert q.stats()["path"] == 3
    q.close()
    sh.close()


# ---------------------------------------------------------------- 4
def test_schema_and_series_churn_after_a_compaction():
    """Column and series indices that move after a compaction: a column that sorts between two names and a sid that sorts into the
    middle; the write is refused while a column has pages in only some of a series' segments, compaction re-cuts that series from
    its first segment, out-of-order rows go into the new column, and the written file reopens with the new sid order."""
    rng = np.random.default_rng(104)
    files = [(_flush(rng, [10, 30, 50], 0, 2600, ("fv", "iv"), 0.0), False)]
    sh = Shard.open_files(_descs(files, seg_rows=700))
    _step_check(sh, files)
    _compact(sh, files, 1000)
    model = _model(files)
    step = {20: _series(T0 + 1000 * SEC + SEC * np.arange(40, dtype=np.int64), _cols(rng, 40, ("fv", "iv"), 0.0))}
    step.update(_after_last(rng, model, [30], 40))
    for s_ in step.values():
        n = s_["times"].size
        s_["cols"]["gv"] = (L.TYPE_FLOAT, rng.normal(7, 1, n), np.ones(n, bool))   # sorts between fv and iv
    _append(sh, files, [(step, False)])
    with pytest.raises(L.OgpuError) as ei:
        write_tssp(sh, "m")
    assert "some of its segments" in str(ei.value)
    plan, _rows = cm.plan(sh.export(), 1000)
    u30 = sh.export()["sids"].tolist().index(30)
    assert (u30, int(sh.export()["series_seg_begin"][u30])) in plan      # from its first segment
    _compact(sh, files, 1000)
    t = T0 + (np.array([1005, 1010.5, 1020, 1500.5, 2000, 2630]) * SEC).astype(np.int64)
    late = {sid: _series(t, {"gv": (L.TYPE_FLOAT, rng.normal(-7, 1, t.size), rng.random(t.size) > 0.2)}) for sid in (20, 30)}
    late[20] = _series(t[:3], {"gv": (L.TYPE_FLOAT, rng.normal(-7, 1, 3), np.ones(3, bool))})
    _append(sh, files, [(late, True)])
    back = Shard.open_tssp(write_tssp(sh, "m"))
    _same_directory_and_pages(sh, back)
    _step_check(back, files)
    back.close(); sh.close()


# ---------------------------------------------------------------- 5
def test_a_written_file_as_the_base_of_a_new_file_set():
    """A shard written partway through its history and reopened holds the same rows; opened as the only ordered file of a new
    shard, it takes the rest of the history's appends as the original does: the same rows at every step, the same directory and
    page bytes after the ordered-only steps."""
    rng = np.random.default_rng(105)
    sids = [2, 4, 6, 8, 10]
    files = [(_flush(rng, sids, 0, 2300, ("fv", "iv"), 0.0), False)]
    sh = Shard.open_files(_descs(files))
    _append(sh, files, [(_late(rng, sids[::2], -100, 2000, 120), True)])
    _append(sh, files, [(_flush(rng, sids, 2300, 500, ("fv", "iv"), 0.0), False)])
    img = write_tssp(sh, "m")
    re = Shard.open_tssp(img)
    _check_rows(re, _model(files))
    re.close()
    other = Shard.open_files([(img, False)])
    _step_check(other, files)
    _same_directory_and_pages(sh, other)
    for step, ordered in (([(_flush(rng, sids, 2800, 300, ("fv", "iv"), 0.0), False)], True),
                          ([(_late(rng, sids[1::2], 1500, 3000, 90), True)], False),
                          ([(_flush(rng, sids + [12], 3100, 200, ("fv", "iv"), 0.0), False)], True)):
        b = dict(step=step, n_rows=other.info()["n_rows"])
        other.append_files(_descs(step))
        _append(sh, files, step)
        _step_check(other, files, b)
        if ordered:
            _same_directory_and_pages(sh, other)
    other.close(); sh.close()


# ---------------------------------------------------------------- 6
def _stored_bytes(files, seg_rows=1000):
    """the page bytes of files as their descriptions hold them"""
    total = 0
    for d, _o in _descs(files, seg_rows=seg_rows):
        for c in range(d.n_columns):
            total += int(np.ctypeslib.as_array(d.columns[c].page_len, shape=(d.n_segments,)).astype(np.int64).sum())
        total += int(np.ctypeslib.as_array(d.time_page_len, shape=(d.n_segments,)).astype(np.int64).sum())
    return total


def test_snappy_pages_through_a_compaction():
    """og_shard_info.page_bytes around Snappy pages (transcoded to raw pages when a file comes in).  The rule, from merge.cu and
    compact.cu: the Snappy counters hold while every transcoded page is in the shard, so page_bytes is the pages as the files
    stored them (Snappy pages at their stored size) until the first append that merges rows or the first compaction that re-cuts
    a series; from then on it is the pages as the shard holds them, later appends included."""
    rng = np.random.default_rng(106)
    n = 2000
    t = T0 + np.arange(n, dtype=np.int64) * SEC
    snappy = {sid: _series(t, {"fv": (L.TYPE_FLOAT, np.round(rng.normal(100, 20, n), 2), np.ones(n, bool)),       # few decimals
                               "iv": (L.TYPE_INT, np.arange(n) * sid, np.ones(n, bool))}) for sid in (1, 2)}
    files = [(snappy, False), (_flush(rng, [1, 2], n, 300, ("fv", "iv"), 0.0), False), (_flush(rng, [1, 2], n + 300, 200, ("fv", "iv"), 0.0), False)]
    sh = Shard.open_files(_descs(files))
    _step_check(sh, files)
    live = int(sh.export()["page_len"].astype(np.int64).sum())
    assert sh.info()["page_bytes"] == _stored_bytes(files) < live                # the Snappy pages as stored
    _compact(sh, files, 1000)                     # the Snappy segments are kept, the tails [300, 200] re-cut
    assert sh.info()["page_bytes"] == int(sh.export()["page_len"].astype(np.int64).sum())
    t2 = t[-1] + SEC * np.arange(600, 1600, dtype=np.int64)
    more = {sid: _series(t2, {"fv": (L.TYPE_FLOAT, np.round(rng.normal(50, 10, t2.size), 2), np.ones(t2.size, bool)),
                              "iv": (L.TYPE_INT, np.arange(t2.size), np.ones(t2.size, bool))}) for sid in (1, 2)}
    _append(sh, files, [(more, False)])
    assert sh.info()["page_bytes"] == int(sh.export()["page_len"].astype(np.int64).sum())
    fresh = Shard.open_files(_descs(files))       # the same files without the compaction: every transcoded page still in it
    assert fresh.info()["page_bytes"] == _stored_bytes(files)
    fresh.close(); sh.close()


# ---------------------------------------------------------------- 7
def test_downsample_mid_history():
    """og_downsample_shard of a shard that went through out-of-order appends and compactions against that of the same rows
    opened as one file: the same sids, rows and cells bit for bit, float sums within n * 2^-53 * sum|x| of the exact sum."""
    rng = np.random.default_rng(107)
    sids = [5, 15, 25, 35, 45, 55]
    files = [(_flush(rng, sids, 0, 2400, ("fv", "iv"), 0.0), False)]
    sh = Shard.open_files(_descs(files, seg_rows=600))
    _compact(sh, files, 1000)
    _append(sh, files, [(_late(rng, sids[::2], -50, 2500, 150), True)])
    _compact(sh, files, 300)
    model = _model(files)
    one = Shard.open_files([(_file_desc(model), False)])
    tmin = min(int(s["times"][0]) for s in model.values())
    tmax = max(int(s["times"][-1]) for s in model.values())
    ops = {L.TYPE_FLOAT: ["sum", "count", "min", "max", "first", "last"], L.TYPE_INT: ["sum", "min", "last"]}
    da, db = sh.downsample_shard(IV, tmin, tmax, ops), one.downsample_shard(IV, tmin, tmax, ops)
    xa, xb = da.open(), db.open()
    ea, eb = xa.export(), xb.export()
    assert np.array_equal(ea["sids"], eb["sids"]) and ea["sids"].tolist() == sorted(model)
    names = [c[0] for c in da.columns()[0]]
    assert names == [c[0] for c in db.columns()[0]]
    wm = ss.window_model(_window_series(model, ["fv", "iv"]), 0, L.TYPE_FLOAT, IV, 0, tmin, tmax, np.arange(len(model)))
    for u in range(ea["sids"].size):
        ra = [xa.decode_segment(g) for g in range(int(ea["series_seg_begin"][u]), int(ea["series_seg_begin"][u + 1]))]
        rb = [xb.decode_segment(g) for g in range(int(eb["series_seg_begin"][u]), int(eb["series_seg_begin"][u + 1]))]
        ta, tb = np.concatenate([r["times"] for r in ra]), np.concatenate([r["times"] for r in rb])
        assert np.array_equal(ta, tb), u
        for c, name in enumerate(names):
            va, vb = np.concatenate([r["cols"][c]["valid"] for r in ra]), np.concatenate([r["cols"][c]["valid"] for r in rb])
            xa_, xb_ = np.concatenate([r["cols"][c]["values"] for r in ra]), np.concatenate([r["cols"][c]["values"] for r in rb])
            assert np.array_equal(va, vb), (u, name)
            if name == "sum_fv":
                cell = u * wm["n_buckets"] + (ta[va] - wm["start"]) // IV
                assert np.all(np.abs(xa_ - xb_) <= 2 * wm["count"][cell] * 2.0**-53 * wm["sum_abs"][cell]), u
                assert np.all(np.abs(xa_ - wm["sum_exact"][cell]) <= wm["count"][cell] * 2.0**-53 * wm["sum_abs"][cell]), u
            else:
                assert np.array_equal(xa_.view(np.uint8), xb_.view(np.uint8)), (u, name)
    xa.close(); xb.close(); da.close(); db.close(); one.close()
    _step_check(sh, files)
    sh.close()


# ---------------------------------------------------------------- 8
def test_a_long_history_leaves_no_device_memory_behind():
    """About forty steps (small ordered flushes, out-of-order files, compactions at changing R, one refusal of each kind): the data
    region holds only live pages after every step, the rows equal the model, and closing the shard returns every buffer."""
    rng = np.random.default_rng(108)
    sids = [1, 2, 3, 4, 5, 6]
    Rs = [7, 1000, 50, 300, 1000, 13, 999, 1000, 1]
    with _NoLeak():
        files = [(_flush(rng, sids, 0, 300, ("fv", "iv"), 0.05), False)]
        sh = Shard.open_files(_descs(files))
        for k in range(36):
            model = _model(files)
            hi = max(int(s["times"][-1]) for s in model.values())
            if k % 4 == 2:
                sh.compact(Rs[k // 4])
            elif k % 4 == 1:
                step = [(_late(rng, sids[k % 3::2], (hi - T0) // SEC - 200, (hi - T0) // SEC + 5, 20), True)]
                sh.append_files(_descs(step)); files += step
            else:
                step = [(_after_last(rng, model, sids if k % 8 == 0 else sids[k % 2::2], 3 + k % 7), False)]
                sh.append_files(_descs(step)); files += step
            assert _data_excess(sh) == 0, k
            if k % 6 == 5:
                _check_rows(sh, _model(files))
        model = _model(files)
        at_last = {1: _series(model[1]["times"][-1:], _cols(rng, 1, ("fv", "iv"), 0.0))}
        wrong_type = {2: _series(model[2]["times"][-1:] + SEC, {"fv": (L.TYPE_INT, np.arange(1), np.ones(1, bool))})}
        q = None
        for call, status in ((lambda: sh.append_files(_descs([(at_last, False)])), L.OG_E_UNSUPPORTED),
                             (lambda: sh.append_files(_descs([(wrong_type, False)])), L.OG_E_TYPE),
                             (lambda: sh.compact(1001), L.OG_E_INVAL),
                             (lambda: sh.append_files(_descs([(_after_last(rng, model, sids, 3), False)])), L.OG_E_STATE),
                             (lambda: sh.compact(7), L.OG_E_STATE)):
            if status == L.OG_E_STATE and q is None:
                q = AggQuery(sh, [("count", 0)], 0, T0, T0 + 9000 * SEC)
            with pytest.raises(L.OgpuError) as ei:
                call()
            assert ei.value.status == status, str(ei.value)
            assert _data_excess(sh) == 0
        q.close()
        sh.compact(1000)
        _step_check(sh, files)
        sh.close()
