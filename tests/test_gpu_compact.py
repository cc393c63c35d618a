"""og_shard_compact: every series of an open shard re-cut into full segments.

The compacted shard must hold exactly what tests/compact_model.py derives from its export before the call (directory and every
page byte), the same rows series by series (og_decode_segment), and answer every query path as the oracle does over its export."""
import numpy as np
import pytest

import compact_model as cm
import oracle
import segment_shards as ss
from opengemini_b200 import AggQuery, Shard, write_tssp
from opengemini_b200 import _lib as L
from test_gpu_append import _dense_equal, _descs, _flush, _late, _same_directory_and_pages
from test_gpu_device_memory import _NoLeak
from test_gpu_out_of_order import SEC, T0, TYPE_STRING, _check_rows, _file_desc, _model, _series

pytestmark = pytest.mark.gpu

COLS = [(L.TYPE_FLOAT, L.SYNTH_F_HI, 0), (L.TYPE_FLOAT, L.SYNTH_F_LO, 50), (L.TYPE_INT, L.SYNTH_INT_WALK, 400), (L.TYPE_BOOL, L.SYNTH_BOOL, 1000)]


@pytest.fixture(scope="module", autouse=True)
def _device():
    Shard.init(0)


def _rows(sh):
    """every series' rows, og_decode_segment over its segments: [(times, [(valid, values)] per column)]"""
    ex = sh.export()
    out = []
    for u in range(ex["sids"].size):
        a, b = int(ex["series_seg_begin"][u]), int(ex["series_seg_begin"][u + 1])
        recs = [sh.decode_segment(g) for g in range(a, b)]
        t = np.concatenate([r["times"] for r in recs])
        cols = [(np.concatenate([r["cols"][c]["valid"] for r in recs]), np.concatenate([r["cols"][c]["values"] for r in recs]).view(np.uint8))
                for c in range(len(recs[0]["cols"]))]
        out.append((t, cols))
    return out


def _same_rows(a, b):
    assert len(a) == len(b)
    for (ta, ca), (tb, cb) in zip(a, b):
        assert np.array_equal(ta, tb)
        for (va, xa), (vb, xb) in zip(ca, cb):
            assert np.array_equal(va, vb) and np.array_equal(xa, xb)


def _compact_as_modelled(sh, R=0):
    """compact `sh` and check it against the model of its export before the call; returns the info"""
    ex = sh.export()
    want = cm.expected(ex, R or 1000)
    rows, info0 = _rows(sh), sh.info()
    info = sh.compact(R)
    got = sh.export()
    cm.assert_matches(got, want)
    assert {k: v for k, v in info.items() if k != "compact_ms"} == want["info"]
    if info["series_rewritten"]:  # the new data region holds the live pages only
        assert got["data"].size == int(got["page_len"].astype(np.int64).sum())
    _same_rows(_rows(sh), rows)
    i1 = sh.info()
    for k in ("n_series", "n_rows", "tmin", "tmax"):
        assert i1[k] == info0[k], k
    assert i1["n_segments"] == got["seg_tmin"].size
    return info


def _against_oracle(sh, ncols):
    """every query path on the compacted shard against the oracle over its export: bitwise in the reference's order, float sums of
    the folded order within 1e-12"""
    ex = sh.export()
    desc = oracle.shard_desc_from_export(ex)
    tmin, tmax = int(ex["seg_tmin"].min()), int(ex["seg_tmax"].max())
    ns = ex["sids"].size
    groups = (np.arange(ns) % 3).astype(np.uint32)
    cases = []
    for c in range(ncols):
        typ = int(ex["col_types"][c])
        calls = [("sum", c), ("count", c), ("max", c)] if typ != L.TYPE_BOOL else [("count", c), ("first", c), ("last", c)]
        cases += [(calls, dict(flags=L.Q_STRICT_ORDER)), (calls, dict(flags=0)), (calls, dict(group="series")),
                  (calls, dict(group="map", series_group=groups, n_groups=3, flags=L.Q_STRICT_ORDER)),
                  (calls, dict(flags=L.Q_STRICT_ORDER, ascending=False))]
    f = [int(t) for t in ex["col_types"][:ncols]].index(L.TYPE_FLOAT)
    if ncols >= 3:  # k_fused_multi
        cases.append(([("sum", f), ("count", (f + 1) % ncols), ("max", f), ("first", (f + 2) % ncols)], dict(flags=L.Q_STRICT_ORDER)))
    cases.append(([("count", f), ("sum", f)], dict(flags=L.Q_STRICT_ORDER, filter=[("term", f, ">", 100.5)])))  # k_fused_cols + WHERE
    for calls, kw in cases:
        q = AggQuery(sh, calls, 60 * SEC, tmin, tmax, **kw).run()
        got = q.dense_host()
        ref = oracle.scan(desc, q.desc, threads=1)
        for k, (f, c) in enumerate(calls):
            rv = ref["cols"][k]["valid"].astype(bool)
            assert np.array_equal(got["cols"][k]["valid"].astype(bool), rv), (calls, kw)
            g, r = got["cols"][k]["values"].view(np.uint64)[rv], ref["cols"][k]["values"][rv]
            if f == "sum" and not (kw.get("flags", 0) & L.Q_STRICT_ORDER) and int(ex["col_types"][c]) == L.TYPE_FLOAT:
                gf, rf = g.view(np.float64), r.view(np.float64)
                with np.errstate(invalid="ignore"):
                    close = (gf == rf) | (np.isnan(gf) & np.isnan(rf)) | (np.abs(gf - rf) <= 1e-12 * np.maximum(1.0, np.abs(rf)))
                assert close.all(), (calls, kw)
            else:
                assert np.array_equal(g, r), (calls, kw)
        q.close()


def _synth_with_flushes(n_series, rows, k, r, R_src=1000, seed=3):
    sh = Shard.synth(n_series, rows, COLS, t0=T0, dt=SEC, seed=seed, rows_per_segment=R_src)
    for i in range(k):
        src = Shard.synth(n_series, r, COLS, t0=T0 + (rows + i * r) * SEC, dt=SEC, seed=seed + 1 + i)
        sh.append_files([(oracle.shard_desc_from_export(src.export()), False)])
        src.close()
    return sh


# ---------------------------------------------------------------- pages and rows against the model, queries against the oracle
@pytest.mark.parametrize("R", [1000, 7, 1])
def test_synth_shard_after_small_flushes(R):
    n_series, rows = (20, 3000) if R != 1 else (4, 300)
    sh = _synth_with_flushes(n_series, rows, 30, 7)
    info = _compact_as_modelled(sh, R)
    assert info["series_rewritten"] == n_series
    _against_oracle(sh, len(COLS))
    assert sh.compact(R)["series_rewritten"] == 0  # a second compaction is a no-op
    sh.close()


@pytest.mark.parametrize("R", [1000, 700])
def test_700_row_synth_shard(R):
    sh = Shard.synth(30, 2500, COLS, t0=T0, dt=SEC, seed=5, rows_per_segment=700)
    ex = sh.export()
    info = _compact_as_modelled(sh, R)
    if R == 700:  # already compact: untouched, every counter zero
        assert all(v == 0 for v in info.values())
        got = sh.export()
        for k in ex:
            assert np.array_equal(ex[k], got[k]), k
    else:
        assert info["series_rewritten"] == 30 and info["segments_kept"] == 0
    _against_oracle(sh, len(COLS))
    sh.close()


def test_merged_shard():
    rng = np.random.default_rng(11)
    sids = [100 + s for s in range(12)]
    files = [(_flush(rng, sids, 0, 2600), False), (_late(rng, sids[::3], -200, 2500, 200), True),
             (_flush(rng, sids, 2600, 30), False), (_flush(rng, sids, 2630, 5), False)]
    sh = Shard.open_files(_descs(files))
    for step in ([(_flush(rng, sids, 2635, 3), False)], [(_late(rng, sids[1::4], 1000, 2600, 50), True)]):
        sh.append_files(_descs(step))
        files += step
    mi = sh.merge_info()
    _compact_as_modelled(sh)
    assert sh.merge_info() == mi  # og_shard_merge_info is not touched
    _check_rows(sh, _model(files))
    _against_oracle(sh, 3)
    sh.close()


def test_infinities_take_the_raw_page_and_nan_rows_survive():
    rng = np.random.default_rng(2)
    rows = ss.series_rows(rng, 1300, ["f_hi", "i_s8b"])
    rows["cols"][0][0][100] = np.inf
    rows["cols"][0][0][800] = -np.inf                       # one new 1000-row segment holds both: raw page
    sh, _d = ss.open_shard([rows], ss.types_of(["f_hi", "i_s8b"]), [[600, 600, 100]])
    _compact_as_modelled(sh)
    _against_oracle(sh, 2)
    sh.close()
    rows["cols"][0][0][5] = np.nan                          # NaN: rows bit for bit
    sh, _d = ss.open_shard([rows], ss.types_of(["f_hi", "i_s8b"]), [[600, 600, 100]])
    before = _rows(sh)
    sh.compact()
    _same_rows(_rows(sh), before)
    sh.close()


# ---------------------------------------------------------------- layout the other entry points rely on
def test_identical_flushes_restore_the_folded_path():
    cols = [(L.TYPE_FLOAT, L.SYNTH_F_HI, 0)]
    sh = Shard.synth(300, 2000, cols, t0=T0, dt=SEC, seed=3)
    for i in range(8):
        src = Shard.synth(300, 125, cols, t0=T0 + (2000 + 125 * i) * SEC, dt=SEC, seed=10 + i)
        sh.append_files([(oracle.shard_desc_from_export(src.export()), False)])
        src.close()
    info = sh.compact()
    assert info["series_rewritten"] == 300 and info["segments_kept"] == 600
    q = AggQuery(sh, [("sum", 0), ("count", 0), ("max", 0)], 60 * SEC, T0, T0 + 2999 * SEC).run()
    assert q.stats()["path"] == 3
    q.close()
    _against_oracle(sh, 1)
    sh.close()


def test_a_shard_with_a_column_from_a_later_flush_becomes_writable():
    rng = np.random.default_rng(1)
    files = [(_flush(rng, [20, 30, 40], 0, 2600), False)]
    step = [(_flush(rng, [25, 40], 2600, 30), False)]
    for s_ in step[0][0].values():
        s_["cols"]["zz"] = (L.TYPE_INT, np.arange(s_["times"].size), np.ones(s_["times"].size, bool))
    sh = Shard.open_files(_descs(files))
    sh.append_files(_descs(step))
    files += step
    with pytest.raises(L.OgpuError) as ei:
        write_tssp(sh, "m")
    assert "some of its segments" in str(ei.value)
    _compact_as_modelled(sh)
    _check_rows(sh, _model(files))
    back = Shard.open_tssp(write_tssp(sh, "m"))
    _same_directory_and_pages(sh, back)
    for c in range(4):
        for calls in ([("count", c)], [("first", c), ("last", c)]):
            _dense_equal(sh, back, calls, 60 * SEC, T0, T0 + 3000 * SEC, flags=L.Q_STRICT_ORDER)
            _dense_equal(sh, back, calls, 60 * SEC, T0, T0 + 3000 * SEC, group="series")
    back.close(); sh.close()


def test_a_segment_longer_than_65536_rows_serves_descending_decode():
    rng = np.random.default_rng(4)
    rows = ss.series_rows(rng, 70000, ["f_hi"])
    sh, _d = ss.open_shard([rows], ss.types_of(["f_hi"]), [[70000]])
    with pytest.raises(L.OgpuError):
        sh.decode_segment(0, descending=True)
    _compact_as_modelled(sh)
    assert sh.info()["n_segments"] == 70
    for g in (0, 69):
        rec = sh.decode_segment(g, descending=True)
        assert np.array_equal(rec["times"], rows["times"][g * 1000:(g + 1) * 1000][::-1])
    sh.close()


# ---------------------------------------------------------------- refusals
def _unchanged(sh, ex, info):
    got = sh.export()
    for k in ex:
        assert np.array_equal(got[k], ex[k]), k
    assert sh.info() == info


def test_refusals_leave_the_shard_as_it_was():
    n = 1200
    t = T0 + np.arange(n, dtype=np.int64) * SEC
    ok = np.ones(n, bool)
    base = {1: _series(t, {"v": (L.TYPE_FLOAT, np.arange(n, dtype=np.float64), ok), "s": (TYPE_STRING, None, ok)}),
            2: _series(t, {"v": (L.TYPE_FLOAT, np.arange(n, dtype=np.float64), ok), "s": (TYPE_STRING, None, ~ok)})}
    sh = Shard.open_files([(_file_desc(base, seg_rows=700), False)])
    ex, info = sh.export(), sh.info()

    def refused(status, text, **kw):
        with pytest.raises(L.OgpuError) as ei:
            sh.compact(**kw)
        assert ei.value.status == status, str(ei.value)
        assert text in str(ei.value), str(ei.value)
        _unchanged(sh, ex, info)

    refused(L.OG_E_UNSUPPORTED, "sid 1", rows_per_segment=1000)      # string values in a re-cut range
    refused(L.OG_E_INVAL, "rows_per_segment", rows_per_segment=1001)
    d, i = L.CompactDesc(0, 1), L.CompactInfo()
    assert L.lib().og_shard_compact(sh.h, d, i) == L.OG_E_INVAL
    q = AggQuery(sh, [("count", 1)], 0, T0, T0 + 2 * n * SEC)
    refused(L.OG_E_STATE, "queries", rows_per_segment=1000)
    q.close()
    assert sh.compact(700)["series_rewritten"] == 0                  # compact at R = 700 already
    sh.close()
    # the all-null string column of sid 2 is fine: an all-null page in every new segment
    sh = Shard.open_files([(_file_desc({2: base[2]}, seg_rows=700), False)])
    want, n_rows = cm.expected(sh.export(), 1000), sh.info()["n_rows"]
    assert sh.compact()["series_rewritten"] == 1
    cm.assert_matches(sh.export(), want)
    assert sh.info()["n_rows"] == n_rows
    q = AggQuery(sh, [("count", 0), ("count", 1)], 0, T0, T0 + 2 * n * SEC, flags=L.Q_STRICT_ORDER).run()
    assert [c["values"].tolist() for c in q.dense_host()["cols"]] == [[0], [n]]
    q.close()
    sh.close()
    # a time repeated in a re-cut range: og_shard_open refuses it across two segments (their time ranges must not touch) and takes
    # it inside one, where compaction finds it
    rows = ss.series_rows(np.random.default_rng(3), 1500, ["f_hi"])
    rows["times"][701] = rows["times"][700]
    d = ss.shard_desc([rows], ss.types_of(["f_hi"]), [[700, 800]])
    sh = Shard.open_desc(d, keepalive=d)
    ex, info = sh.export(), sh.info()
    refused(L.OG_E_CORRUPT, str(int(rows["times"][701])))
    sh.close()


# ---------------------------------------------------------------- batches and device memory
def test_batches_give_the_same_bytes(monkeypatch):
    a = _synth_with_flushes(12, 2500, 10, 13, seed=8)
    b = _synth_with_flushes(12, 2500, 10, 13, seed=8)
    a.compact()
    monkeypatch.setenv("OGPU_COMPACT_BATCH_ROWS", "1500")
    b.compact()
    ea, eb = a.export(), b.export()
    for k in ("sids", "series_seg_begin", "seg_tmin", "seg_tmax", "page_len"):
        assert np.array_equal(ea[k], eb[k]), k
    _same_directory_and_pages(a, b)
    a.close(); b.close()


def test_no_device_memory_is_left_behind():
    with _NoLeak():
        sh = _synth_with_flushes(16, 2000, 3, 9, seed=4)
        for r in (7, 1000, 1000, 300):
            sh.compact(r)
        with pytest.raises(L.OgpuError):
            sh.compact(1001)
        sh.close()
    sh = _synth_with_flushes(16, 2000, 3, 9, seed=4)
    sh.compact()
    with _NoLeak():  # a compaction of a compact shard allocates nothing it keeps
        sh.compact()
    sh.close()
