"""og_shard_append_files: files flushed after a shard was built, added to the open shard.

After every append the shard must answer as og_shard_open_files over all of its files would: the rows of every series bit for bit
(og_decode_segment), og_shard_info, every query path against scan_aggregate_files (tests/oracle_files.py), TSSP write and
downsample.  Ordered-only appends keep the directory and page bytes of the fresh open as well."""
import numpy as np
import pytest

import oracle
import oracle_files
from opengemini_b200 import AggQuery, Shard, write_tssp
from opengemini_b200 import _lib as L
from test_gpu_out_of_order import ALL6, SEC, T0, TYPE_STRING, _check_rows, _file_desc, _model, _series

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module", autouse=True)
def _device():
    Shard.init(0)


def _cols(rng, n, present=("fv", "iv", "bv"), null_p=0.05):
    c = {}
    if "fv" in present:
        c["fv"] = (L.TYPE_FLOAT, np.round(rng.normal(100, 20, n), 3) + rng.random(n) * 1e-6, rng.random(n) >= null_p)
    if "iv" in present:
        c["iv"] = (L.TYPE_INT, rng.integers(-1000, 1000, n).cumsum(), rng.random(n) >= null_p)
    if "bv" in present:
        c["bv"] = (L.TYPE_BOOL, (rng.random(n) < 0.5).astype(np.uint8), rng.random(n) >= null_p)
    return c


def _flush(rng, sids, t_lo, n, present=("fv", "iv", "bv"), null_p=0.05):
    t = T0 + (t_lo + np.arange(n, dtype=np.int64)) * SEC
    return {sid: _series(t, _cols(rng, n, present, null_p)) for sid in sids}


def _late(rng, sids, t_lo, t_hi, k, present=("fv", "iv")):
    out = {}
    for sid in sids:
        t = np.unique(T0 + rng.integers(t_lo, t_hi, k) * SEC + np.where(rng.random(k) < 0.3, SEC // 2, 0))
        out[sid] = _series(t, _cols(rng, t.size, present, 0.2))
    return out


def _descs(files, **kw):
    return [(_file_desc(f, **kw), ooo) for f, ooo in files]


def _same_directory_and_pages(a, b):
    ea, eb = a.export(), b.export()
    for k in ("sids", "series_seg_begin", "seg_tmin", "seg_tmax", "page_len", "col_types"):
        assert np.array_equal(ea[k], eb[k]), k
    for c in range(ea["page_off"].shape[0]):
        for g in range(ea["seg_tmin"].size):
            la = int(ea["page_len"][c][g])
            oa, ob = int(ea["page_off"][c][g]), int(eb["page_off"][c][g])
            assert np.array_equal(ea["data"][oa:oa + la], eb["data"][ob:ob + la]), (c, g)


def _dense_equal(a, b, calls, iv, tmin, tmax, **kw):
    qa = AggQuery(a, calls, iv, tmin, tmax, **kw).run()
    qb = AggQuery(b, calls, iv, tmin, tmax, **kw).run()
    da, db = qa.dense_host(), qb.dense_host()
    for k in range(len(calls)):
        assert np.array_equal(da["cols"][k]["valid"], db["cols"][k]["valid"]), (calls, kw)
        assert np.array_equal(da["cols"][k]["values"].view(np.uint64), db["cols"][k]["values"].view(np.uint64)), (calls, kw)
    pa, pb = qa.stats()["path"], qb.stats()["path"]
    qa.close(); qb.close()
    assert pa == pb, (calls, kw, pa, pb)
    return pa


def _data_excess(sh):
    ex = sh.export()
    return ex["data"].size - int(ex["page_len"].astype(np.int64).sum())


def _compare(sh, files, calls, iv, tmin, tmax, where=None, seg_rows=1000, **kw):
    """The query on the shard against scan_aggregate_files over the whole file set, as test_gpu_out_of_order.py compares:
    bitwise, except float sums of groups that hold a series with out-of-order rows (1e-12 relative)."""
    names = sorted({n for f, _ in files for s_ in f.values() for n in s_["cols"]})
    flt = [(it if it in ("and", "or") else ("term", it[0], it[1], it[2])) for it in where] if where else None
    flt_named = [(it if it in ("and", "or") else (names[it[0]], it[1], it[2])) for it in where] if where else None
    q = AggQuery(sh, calls, iv, tmin, tmax, filter=flt, **kw).run()
    got = q.dense_host()
    ref, sids = oracle_files.scan_aggregate_files(files, q, flt_named, seg_rows=seg_rows)
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
    q.close()


def _all_paths(sh, files, seg_rows=1000):
    """every query path against the restated file-set read over the whole set"""
    model = _model(files)
    names = sorted({n for f, _ in files for s_ in f.values() for n in s_["cols"]})
    fv, iv_ = names.index("fv"), names.index("iv")
    tmin = min(int(s["times"][0]) for s in model.values())
    tmax = max(int(s["times"][-1]) for s in model.values())
    groups = np.arange(len(model), dtype=np.uint32) % 3
    for calls in ([("sum", fv), ("count", fv), ("max", fv)], [(f, fv) for f in ALL6], [("min", iv_), ("sum", iv_), ("last", iv_)]):
        _compare(sh, files, calls, 60 * SEC, tmin, tmax, seg_rows=seg_rows, flags=L.Q_STRICT_ORDER)
        _compare(sh, files, calls, 60 * SEC, tmin, tmax, seg_rows=seg_rows, flags=0)
        _compare(sh, files, calls, 60 * SEC, tmin, tmax, seg_rows=seg_rows, group="series")
        _compare(sh, files, calls, 45 * SEC, tmin, tmax, seg_rows=seg_rows, group="map", series_group=groups, n_groups=3)
        _compare(sh, files, calls, 60 * SEC, tmin, tmax, seg_rows=seg_rows, flags=L.Q_NO_FUSED | L.Q_STRICT_ORDER)
    _compare(sh, files, [("sum", iv_), ("count", fv), ("max", fv), ("first", iv_)], 60 * SEC, tmin, tmax, seg_rows=seg_rows,
             flags=L.Q_STRICT_ORDER)  # k_fused_multi
    thr = float(np.median(np.concatenate([s_["cols"]["fv"][1] for f, _ in files for s_ in f.values() if "fv" in s_["cols"]])))
    if not any(ooo for _f, ooo in files):
        _compare(sh, files, [("count", fv), ("sum", fv)], 60 * SEC, tmin, tmax, where=[(fv, ">", thr)], seg_rows=seg_rows,
                 flags=L.Q_STRICT_ORDER)  # k_fused_cols + WHERE
        _compare(sh, files, [("count", fv), ("sum", iv_)], 60 * SEC, tmin, tmax, where=[(iv_, "<", 0)], seg_rows=seg_rows, group="series")
        return
    # WHERE applies to the merged row, the reference filters each file first (DESIGN.md "Deviations"): against the fresh open
    fresh = Shard.open_files(_descs(files, seg_rows=seg_rows))
    for where, group in (([("term", fv, ">", thr)], "all"), ([("term", iv_, "<", 0)], "series")):
        qa = AggQuery(sh, [("count", fv), ("count", iv_)], 60 * SEC, tmin, tmax, filter=where, group=group, flags=L.Q_STRICT_ORDER).run()
        qb = AggQuery(fresh, [("count", fv), ("count", iv_)], 60 * SEC, tmin, tmax, filter=where, group=group, flags=L.Q_STRICT_ORDER).run()
        for ca, cb in zip(qa.dense_host()["cols"], qb.dense_host()["cols"]):
            assert np.array_equal(ca["valid"], cb["valid"]) and np.array_equal(ca["values"], cb["values"]), where
        qa.close(); qb.close()
    fresh.close()


def _info_like(sh, fresh, ordered_only):
    a, b = sh.info(), fresh.info()
    if not ordered_only:  # re-encoded spans may be cut into different segments: rows and range still agree
        for k in ("n_segments", "page_bytes"):
            a.pop(k); b.pop(k)
    assert a == b


# ---------------------------------------------------------------- ordered flushes
def test_ordered_appends_equal_the_fresh_open():
    rng = np.random.default_rng(1)
    files = [(_flush(rng, [20, 30, 40], 0, 2600), False)]
    sh = Shard.open_files(_descs(files))
    steps = [
        [(_flush(rng, [10, 30, 40], 2600, 1500, present=("fv", "iv")), False)],           # sid first, no bool column
        [(_flush(rng, [25, 40, 50], 4100, 1200), False),                                  # sids between and last
         (_flush(rng, [10, 20], 5300, 700), False)],                                       # two files in one call
    ]
    for s_ in steps[1][0][0].values():  # a new integer column that sorts last
        s_["cols"]["zz"] = (L.TYPE_INT, np.arange(s_["times"].size), np.ones(s_["times"].size, bool))
    for step in steps:
        sh.append_files(_descs(step))
        files += step
        fresh = Shard.open_files(_descs(files))
        _same_directory_and_pages(sh, fresh)
        _info_like(sh, fresh, True)
        _check_rows(sh, _model(files))
        assert _data_excess(sh) == 0  # the live pages only
        mi = sh.merge_info()
        assert mi["n_files"] == len(step) and mi["n_out_of_order_files"] == 0 and mi["segments_rewritten_out"] == 0
        names = sorted({n for f, _ in files for s_ in f.values() for n in s_["cols"]})
        fv = names.index("fv")
        for calls in ([("sum", fv), ("count", fv), ("max", fv)], [(f, fv) for f in ALL6], [("sum", names.index("iv")), ("min", fv)]):
            for flags in (0, L.Q_STRICT_ORDER, L.Q_NO_FUSED):
                _dense_equal(sh, fresh, calls, 60 * SEC, T0, T0 + 6000 * SEC, flags=flags)
            _dense_equal(sh, fresh, calls, 60 * SEC, T0, T0 + 6000 * SEC, group="series")
        _all_paths(sh, files)
        fresh.close()
    sh.close()


def test_a_regular_synth_shard_keeps_the_folded_path():
    cols = [(L.TYPE_FLOAT, L.SYNTH_F_HI, 0), (L.TYPE_INT, L.SYNTH_INT_WALK, 0)]
    base = Shard.synth(300, 2000, cols, t0=T0, dt=SEC, seed=3)
    ex = base.export()
    flush_src = Shard.synth(300, 1000, cols, t0=T0 + 2000 * SEC, dt=SEC, seed=4)
    flush = oracle.shard_desc_from_export(flush_src.export())
    base.append_files([(flush, False)])
    fresh = Shard.open_files([(oracle.shard_desc_from_export(ex), False), (flush, False)])
    _same_directory_and_pages(base, fresh)
    _info_like(base, fresh, True)
    for calls in ([("sum", 0), ("count", 0), ("max", 0)], [(f, 0) for f in ALL6]):
        assert _dense_equal(base, fresh, calls, 60 * SEC, T0, T0 + 2999 * SEC) == 3
        _dense_equal(base, fresh, calls, 60 * SEC, T0, T0 + 2999 * SEC, flags=L.Q_STRICT_ORDER)
    # the flush arrives while the interleaved copy of the base exists: it is rebuilt for the new layout
    q = AggQuery(base, [("sum", 0)], 60 * SEC, T0, T0 + 2999 * SEC).run(); q.close()
    more = oracle.shard_desc_from_export(Shard.synth(300, 1000, cols, t0=T0 + 3000 * SEC, dt=SEC, seed=5).export())
    base.append_files([(more, False)])
    fresh2 = Shard.open_files([(oracle.shard_desc_from_export(ex), False), (flush, False), (more, False)])
    assert _dense_equal(base, fresh2, [("sum", 0), ("count", 0), ("max", 0)], 60 * SEC, T0, T0 + 3999 * SEC) == 3
    base.close(); fresh.close(); fresh2.close(); flush_src.close()


# ---------------------------------------------------------------- out-of-order flushes
@pytest.mark.parametrize("seg_rows", [1000, 700])
def test_out_of_order_flushes_equal_the_fresh_open(seg_rows):
    rng = np.random.default_rng(seg_rows)
    sids = [100 + s for s in range(12)]
    files = [(_flush(rng, sids, 0, 2600), False), (_late(rng, sids[::3], -200, 2800, 200), True)]
    sh = Shard.open_files(_descs(files, seg_rows=seg_rows))
    # each flush splits its rows at the series' last flushed time: out-of-order files hold only times before it
    steps = [
        [(_flush(rng, sids + [5, 999], 2900, 1800), False),                     # ordered and out-of-order in one call
         (_late(rng, sids[1::4], 1000, 2600, 250, present=("fv", "bv")), True)],
        [(_late(rng, sids[::3], -100, 2700, 150), True)],                         # lands on rows an earlier open merged
        [(_late(rng, sids[1::4] + [5], 2000, 4600, 120), True)],                  # ... and an earlier append merged
        [(_flush(rng, sids, 4700, 800), False),                                   # a span across the shard's last time that
         (_late(rng, sids[::5], 4500, 5300, 100), True)],                         # reaches into the same call's ordered file
    ]
    for step in steps:
        before = sh.info()["n_rows"]
        sh.append_files(_descs(step, seg_rows=seg_rows))
        files += step
        model = _model(files)
        fresh = Shard.open_files(_descs(files, seg_rows=seg_rows))
        _check_rows(sh, model)
        _info_like(sh, fresh, False)
        mi = sh.merge_info()
        assert mi["n_files"] == len(step) and mi["n_out_of_order_files"] == sum(o for _, o in step)
        assert mi["out_of_order_rows"] == sum(s_["times"].size for f, o in step if o for s_ in f.values())
        assert mi["rows_after_merge"] == sh.info()["n_rows"] == sum(s_["times"].size for s_ in model.values())
        assert mi["series_merged"] == len({sid for f, o in step if o for sid in f})
        in_rows = before + sum(s_["times"].size for f, _ in step for s_ in f.values())
        assert mi["rows_replaced"] == in_rows - mi["rows_after_merge"]
        ex = sh.export()
        assert mi["segments_kept"] + mi["segments_rewritten_out"] == ex["seg_tmin"].size
        # the data region holds the live pages only: the pages this call rewrote are left behind
        assert _data_excess(sh) == 0
        assert _data_excess(fresh) == 0
        _all_paths(sh, files, seg_rows)
        fresh.close()
    sh.close()


def test_snappy_pages_in_an_appended_file():
    n = 3000
    t = T0 + np.arange(n, dtype=np.int64) * SEC
    v = np.round(np.linspace(1, 2, n), 1)            # few decimals: the oracle encoder takes Snappy
    base = {7: _series(t[:1500], {"fv": (L.TYPE_FLOAT, v[:1500], np.ones(1500, bool)), "iv": (L.TYPE_INT, np.arange(1500), np.ones(1500, bool))})}
    flush = {7: _series(t[1500:], {"fv": (L.TYPE_FLOAT, v[1500:], np.ones(1500, bool)), "iv": (L.TYPE_INT, np.arange(1500), np.ones(1500, bool))}),
             8: _series(t[1500:], {"fv": (L.TYPE_FLOAT, v[:1500], np.ones(1500, bool)), "iv": (L.TYPE_INT, np.arange(1500), np.ones(1500, bool))})}
    files = [(base, False), (flush, False)]
    sh = Shard.open_files(_descs(files[:1]))
    sh.append_files(_descs(files[1:]))
    fresh = Shard.open_files(_descs(files))
    _same_directory_and_pages(sh, fresh)
    _info_like(sh, fresh, True)
    _check_rows(sh, _model(files))
    late = {8: _series(t[1600:1700:3] + SEC // 2, {"fv": (L.TYPE_FLOAT, np.full(34, 0.5), np.ones(34, bool))})}
    sh.append_files(_descs([(late, True)]))
    files.append((late, True))
    fresh2 = Shard.open_files(_descs(files))
    _check_rows(sh, _model(files))
    _info_like(sh, fresh2, False)
    _all_paths(sh, files)
    sh.close(); fresh.close(); fresh2.close()


# ---------------------------------------------------------------- a downsample result opened in place
def _desc_of_downsampled(ds):
    x = ds.open()
    ex = x.export()
    cols, _t = ds.columns()
    d = Shard.desc(ex["data"], ex["sids"], ex["series_seg_begin"], ex["seg_tmin"], ex["seg_tmax"],
                   [(name, typ, ex["page_off"][c], ex["page_len"][c]) for c, (name, typ, _po, _pl) in enumerate(cols)],
                   ex["page_off"][len(cols)], ex["page_len"][len(cols)])
    x.close()
    return d


def test_a_downsample_result_opened_in_place_as_the_base():
    cols = [(L.TYPE_FLOAT, L.SYNTH_F_HI, 0), (L.TYPE_INT, L.SYNTH_INT_WALK, 0)]
    src = Shard.synth(40, 20000, cols, t0=T0, dt=SEC, seed=9)
    ops = {L.TYPE_FLOAT: ["min", "max", "sum", "count"], L.TYPE_INT: ["sum", "last"]}
    split = T0 + 11980 * SEC  # a window boundary: windows are aligned to the epoch
    da = src.downsample_shard(60 * SEC, T0, split - 1, ops)
    db = src.downsample_shard(60 * SEC, split, T0 + 20000 * SEC, ops)
    caller_bytes = da.export().copy()
    desc_a, desc_b = _desc_of_downsampled(da), _desc_of_downsampled(db)
    base = da.open()
    base.append_files([(desc_b, False)])
    assert np.array_equal(da.export(), caller_bytes)  # the caller's buffer is never written
    fresh = Shard.open_files([(desc_a, False), (desc_b, False)])
    _same_directory_and_pages(base, fresh)
    _info_like(base, fresh, True)
    nc = fresh.export()["col_types"].size
    for c in range(nc):
        for calls in ([("sum", c), ("count", c)], [("max", c), ("first", c), ("last", c)]):
            _dense_equal(base, fresh, calls, 600 * SEC, T0, T0 + 20000 * SEC, flags=L.Q_STRICT_ORDER)
            _dense_equal(base, fresh, calls, 600 * SEC, T0, T0 + 20000 * SEC, group="series")
    base.close(); fresh.close(); da.close(); db.close(); src.close()


# ---------------------------------------------------------------- write and downsample after an append
def test_write_tssp_and_downsample_of_an_appended_shard():
    rng = np.random.default_rng(21)
    sids = [3, 9, 14]
    files = [(_flush(rng, sids, 0, 2500, present=("fv", "iv"), null_p=0.0), False)]
    sh = Shard.open_files(_descs(files))
    step = [(_flush(rng, [1] + sids, 2500, 1500, present=("fv", "iv"), null_p=0.0), False),
            (_late(rng, sids[:2], 100, 3900, 300), True)]
    sh.append_files(_descs(step))
    files += step
    fresh = Shard.open_files(_descs(files))
    # the same rows in (possibly) different segments: the reopened files must hold the same rows
    fa, fb = Shard.open_tssp(write_tssp(sh, "m")), Shard.open_tssp(write_tssp(fresh, "m"))
    _check_rows(fa, _model(files)); _check_rows(fb, _model(files))
    fa.close(); fb.close()
    ops = {L.TYPE_FLOAT: ["min", "max", "count", "first", "last"], L.TYPE_INT: ["sum", "count"]}
    xa = sh.downsample_shard(60 * SEC, T0, T0 + 4000 * SEC, ops).open()
    xb = fresh.downsample_shard(60 * SEC, T0, T0 + 4000 * SEC, ops).open()
    ea, eb = xa.export(), xb.export()
    assert np.array_equal(ea["sids"], eb["sids"]) and np.array_equal(ea["series_seg_begin"], eb["series_seg_begin"])
    for c in range(ea["col_types"].size):
        _dense_equal(xa, xb, [("max", c), ("count", c)], 0, T0 - 60 * SEC, T0 + 4000 * SEC, group="series", flags=L.Q_STRICT_ORDER)
    xa.close(); xb.close()
    # ordered-only: the written file is byte for byte that of the fresh open
    more = [(_flush(rng, sids, 4000, 1000, present=("fv", "iv"), null_p=0.0), False)]
    sh2 = Shard.open_files(_descs(files[:1]))
    sh2.append_files(_descs(more))
    fresh2 = Shard.open_files(_descs(files[:1] + more))
    assert write_tssp(sh2, "m") == write_tssp(fresh2, "m")
    sh2.close(); fresh2.close(); sh.close(); fresh.close()


# ---------------------------------------------------------------- refusals
def _snapshot(sh, col=1):
    q = AggQuery(sh, [("sum", col), ("count", col), ("max", col)], 60 * SEC, T0 - 1000 * SEC, T0 + 9000 * SEC, group="series", flags=L.Q_STRICT_ORDER).run()
    d = q.dense_host()
    q.close()
    return sh.export(), sh.info(), [(c["valid"].copy(), c["values"].view(np.uint64).copy()) for c in d["cols"]]


def _unchanged(sh, snap):
    ex, info, dense = _snapshot(sh)
    for k in ex:
        assert np.array_equal(ex[k], snap[0][k]), k
    assert info == snap[1]
    for (va, xa), (vb, xb) in zip(dense, snap[2]):
        assert np.array_equal(va, vb) and np.array_equal(xa, xb)


def test_refusals_leave_the_shard_as_it_was():
    n = 1200
    t = T0 + np.arange(n, dtype=np.int64) * SEC
    ok = np.ones(n, bool)
    base = {1: _series(t, {"v": (L.TYPE_FLOAT, np.arange(n, dtype=np.float64), ok), "s": (TYPE_STRING, None, ok)}),
            2: _series(t, {"v": (L.TYPE_FLOAT, np.arange(n, dtype=np.float64), ok)})}
    sh = Shard.open_files(_descs([(base, False)]))
    snap = _snapshot(sh)
    tn = t[-1] + SEC * np.arange(1, 11)

    def refused(files, status, text=None):
        with pytest.raises(L.OgpuError) as ei:
            sh.append_files(files)
        assert ei.value.status == status, str(ei.value)
        if text:
            assert text in str(ei.value), str(ei.value)
        _unchanged(sh, snap)

    refused(_descs([({2: _series(tn, {"v": (L.TYPE_INT, np.arange(10), np.ones(10, bool))})}, False)]), L.OG_E_TYPE, '"v"')
    refused(_descs([({2: _series(t[-5:], {"v": (L.TYPE_FLOAT, np.ones(5), np.ones(5, bool))})}, False)]), L.OG_E_UNSUPPORTED, "sid 2")  # flush rule
    refused(_descs([({1: _series(t[5:6] + 1, {"v": (L.TYPE_FLOAT, np.array([1.5]), np.ones(1, bool))})}, True)]), L.OG_E_UNSUPPORTED, '"s"')
    tl = np.array([t[3] + 1, t[3] + 1, t[4] + 1], np.int64)
    refused(_descs([({2: _series(tl, {"v": (L.TYPE_FLOAT, np.array([1.0, 2.0, 3.0]), np.ones(3, bool))})}, True)]), L.OG_E_CORRUPT, "twice")
    good = _file_desc({2: _series(tn, {"v": (L.TYPE_FLOAT, np.arange(10.0), np.ones(10, bool))})})
    dev = _file_desc({2: _series(tn, {"v": (L.TYPE_FLOAT, np.arange(10.0), np.ones(10, bool))})})
    dev.flags = L.SHARD_DEVICE_DATA
    refused([(dev, False)], L.OG_E_INVAL, "OG_SHARD_DEVICE_DATA")
    bad = _file_desc({2: _series(tn, {"v": (L.TYPE_FLOAT, np.arange(10.0), np.ones(10, bool))})})
    np.ctypeslib.as_array(bad.data, shape=(bad.data_len,))[:] = 0xEE  # every page corrupt
    with pytest.raises(L.OgpuError) as ei:
        sh.append_files([(bad, False)])
    assert ei.value.status in (L.OG_E_CORRUPT, L.OG_E_UNSUPPORTED)
    _unchanged(sh, snap)
    q = AggQuery(sh, [("count", 0)], 0, T0, T0 + 2 * n * SEC)
    refused([(good, False)], L.OG_E_STATE, "queries")
    q.close()
    sh.append_files([(good, False)])  # a valid append after every refusal
    q = AggQuery(sh, [("count", 1)], 0, T0, T0 + 2 * n * SEC, group="series", flags=L.Q_STRICT_ORDER).run()
    assert q.dense_host()["cols"][0]["values"].tolist() == [n, n + 10]
    sh.close()
    q.close()  # a query of a closed shard may still be destroyed
