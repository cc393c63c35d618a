"""og_shard_append_rows / og_shard_open_rows at their edges and inside shard histories.

Every flush is checked as test_gpu_append_rows.py checks one: against og_shard_append_files of the two files tests/flush_model.py
writes for the same rows, on a twin shard that goes through the same history (directory, every page byte, og_shard_info and
og_shard_merge_info), and row by row against the merged model of every file so far.  Inside a history, _step_check
(test_gpu_shard_history.py) also runs every aggregate path against the window model and the oracle after every step.

  seeded memtables   1-300 series, sids before, between and after the shard's, 1-20 000 rows each, repeated and shuffled,
                     per-series column subsets, null ratios 0 / 5 / 40 / 100 %, late fractions 0 / 1 / 50 / 100 %
  expand edges       k_flush_expand's 8192-row chunks: series of 8191 ... 16 385 rows, bitmap offsets up to 63, nulls on chunk
                     edges, an all-null chunk before a full one, float, int and bool columns
  time and value     every time page form, times near the int64 limits, one time repeated, ints at the limits and with deltas
                     past 2^60 (raw pages), +Inf with -Inf, a column null throughout one part or the whole record
  histories          flushes between compactions, out-of-order files, a TSSP write, Snappy pages and a downsample"""
import numpy as np
import pytest

import compact_model as cm
import flush_model as fm
import page_forms as pf
from opengemini_b200 import AggQuery, Shard, write_tssp
from opengemini_b200 import _lib as L
from test_gpu_append import _all_paths, _cols, _data_excess, _same_directory_and_pages
from test_gpu_append_rows import _descs, _same_merge_info, _shuffle_and_repeat, _Twins
from test_gpu_device_memory import _NoLeak
from test_gpu_out_of_order import SEC, T0, _check_rows, _file_desc, _model, _series
from test_gpu_shard_history import IV, _step_check

pytestmark = pytest.mark.gpu
I64_MIN, I64_MAX = pf.I64_MIN, pf.I64_MAX
S8B_MAX = (1 << 60) - 1


@pytest.fixture(scope="module", autouse=True)
def _device():
    Shard.init(0)


def _twins_of_rows(batch):
    """_Twins whose shard is og_shard_open_rows of batch and whose twin opens the model's files"""
    tw = _Twins.__new__(_Twins)
    tw.files = fm.files(batch)
    tw.sh, tw.tw = Shard.open_rows(batch), Shard.open_files(_descs(tw.files))
    _twin_check(tw.sh, tw.tw, tw.files)
    return tw


def _column_pages(sh, sid, c):
    """the pages column c holds in the segments of series sid"""
    ex = sh.export()
    u = ex["sids"].tolist().index(sid)
    return [ex["data"][int(ex["page_off"][c][g]):int(ex["page_off"][c][g]) + int(ex["page_len"][c][g])]
            for g in range(int(ex["series_seg_begin"][u]), int(ex["series_seg_begin"][u + 1])) if ex["page_len"][c][g]]


def _twin_check(sh, tw, files):
    _same_directory_and_pages(sh, tw)
    assert sh.info() == tw.info()
    _same_merge_info(sh, tw)
    _check_rows(sh, _model(files))


# ---------------------------------------------------------------- seeded memtables
def _memtable(rng, model, budget):
    """one flush: {sid: series} in arrival order; model: the shard's rows so far (sids, last times)"""
    held = sorted(model)
    lo_sid, hi_sid = held[0], held[-1]
    n_ser = int(min(300, max(1, np.exp(rng.uniform(0, np.log(300))))))
    pool = set(rng.choice(held, min(len(held), n_ser), replace=False).tolist())
    pool |= {int(x) for x in rng.integers(1, lo_sid + 1, 3)} | {int(x) for x in rng.integers(lo_sid, hi_sid + 1, n_ser // 3 + 1)}
    pool |= {hi_sid + int(x) for x in rng.integers(1, 1000, 3)}
    sids = sorted(pool)[:n_ser] if len(pool) > n_ser else sorted(pool)
    per = max(1, budget // len(sids))
    out = {}
    for sid in sids:
        n = int(min(per, max(1, np.exp(rng.uniform(0, np.log(20000))))))
        late = [0.0, 0.01, 0.5, 1.0][int(rng.integers(0, 4))] if sid in model else 0.0
        k_late = int(round(n * late))
        last = int(model[sid]["times"][-1]) if sid in model else T0
        first = int(model[sid]["times"][0]) if sid in model else T0
        t_new = last + SEC * (1 + np.arange(n - k_late, dtype=np.int64)) * int(rng.integers(1, 3))
        t_late = np.unique(first - 20 * SEC + rng.integers(0, max(1, (last - first) // (SEC // 2) + 41), k_late) * (SEC // 2))
        t_late = t_late[t_late <= last]
        t = np.concatenate([t_new, t_late]).astype(np.int64)
        present = [c for c in ("fv", "iv", "bv") if rng.random() < 0.7] or ["fv"]
        cols = {}
        for c in present:
            null_p = [0.0, 0.05, 0.4, 1.0][int(rng.integers(0, 4))]
            cols.update(_cols(rng, t.size, (c,), null_p))
        out[sid] = _series(t, cols)
    return _shuffle_and_repeat(rng, out, int(rng.integers(1, 6)))


@pytest.mark.parametrize("seed", range(30))
def test_seeded_memtables(seed):
    rng = np.random.default_rng(1000 + seed)
    base_sids = sorted({int(x) for x in rng.integers(50, 5000, int(rng.integers(1, 40)))})
    n0 = int(rng.integers(1, 2500))
    base = {sid: _series(T0 + np.arange(n0, dtype=np.int64) * SEC, _cols(rng, n0, ("fv", "iv", "bv"), 0.05)) for sid in base_sids}
    tw = _Twins([(base, False)])
    for k in range(int(rng.integers(2, 4))):
        batch = _memtable(rng, _model(tw.files), budget=int(rng.integers(2000, 40000)))
        tw.flush(batch, paths=(seed + k) % 4 == 0)  # every aggregate path on a rotating quarter of the flushes
    tw.close()


# ---------------------------------------------------------------- k_flush_expand chunk edges
@pytest.mark.parametrize("n", [8191, 8192, 8193, 16384, 16385])
def test_expand_chunk_edges(n):
    """one series of n rows in arrival order, three columns at bitmap offsets (0, 1, 7) then (8, 9, 63): nulls on the first and
    last row of every 8192-row chunk, and (n > 8192) the float column null through the whole first chunk and valid through the
    second; then late rows, so both parts are written"""
    rng = np.random.default_rng(n)
    tw = _Twins([(fm.flush({3: _series(T0 + np.arange(500, dtype=np.int64) * SEC, _cols(rng, 500, ("fv", "iv", "bv"), 0.1))})[0], False)])
    t0 = 500
    for offs in ((0, 1, 7), (8, 9, 63)):
        t = np.concatenate([T0 + (t0 + np.arange(n, dtype=np.int64)) * SEC, T0 + np.arange(0, 400, 7, dtype=np.int64) * SEC + SEC // 2])
        m = t.size
        edges = sorted({e for c in range(0, m, 8192) for e in (c, min(c + 8191, m - 1))} | {m - 1})
        cols = {}
        for name, c in _cols(rng, m, ("bv", "fv", "iv"), 0.05).items():
            ok = c[2].copy()
            ok[edges] = False
            cols[name] = (c[0], c[1], ok)
        fv_ok = cols["fv"][2]
        if n > 8192:
            fv_ok[:8192] = False; fv_ok[8192:16384] = True
        cols["bv"][2][edges[:2]] = True  # the bool column valid on the first chunk's edges
        batch = {3: _series(t, cols)}
        d = Shard.rows_desc([(nm, cols[nm][0]) for nm in ("bv", "fv", "iv")],
                            [(3, t, [Shard.colval(*cols[nm], bitmap_offset=o) for nm, o in zip(("bv", "fv", "iv"), offs)])])
        new = fm.files(batch, fm.last_times(tw.tw.export()))
        assert [o for _f, o in new] == [False, True]
        tw.sh.append_rows(d)
        tw.tw.append_files(_descs(new))
        tw.files += new
        _twin_check(tw.sh, tw.tw, tw.files)
        t0 += n
    _all_paths(tw.sh, tw.files)
    tw.close()


# ---------------------------------------------------------------- time and value edges
def _time_forms():
    """{sid: times}: a series per time page form a flush can write (segments of 1000 rows from each part's first row)"""
    rng = np.random.default_rng(31)
    n = 2300
    f = {1: T0 + np.arange(n, dtype=np.int64) * SEC,                                                  # const
         2: T0 + np.cumsum(rng.integers(1, 40, n) * 10),                                              # multiples of 10: scale 1
         3: T0 + np.cumsum(rng.integers(1, 9, n)),                                                    # scale 1
         4: -(10**15) + np.cumsum(rng.integers(1, 99, n) * 1000),                                     # negative, scale 1000
         5: -(10**12) + np.cumsum(rng.integers(1, 5, n) * 10**6)}                                     # crosses 0, scale 10^6
    for k in (2, 3, 4, 5, 7, 8):
        f[10 + k] = T0 + np.cumsum(rng.integers(1, 30, n) * 10**k)                                    # scale 10^k
    # raw time pages: one delta of 2^60 - 1 or more in a segment, the rest random (Snappy would not shrink them)
    t = -(1 << 62) + np.cumsum(rng.integers(1, 1 << 40, n)).astype(np.int64)
    t[1500:] += S8B_MAX
    f[30] = t
    t = -(1 << 62) + np.cumsum(rng.integers(1, 1 << 40, n)).astype(np.int64)
    t[700:] += S8B_MAX - 1 - int(t[700] - t[699])                                                      # one delta of 2^60 - 2: Simple8b
    f[31] = t
    t = np.cumsum(rng.integers(1, 1 << 40, 900)).astype(np.int64)
    t[400:] += S8B_MAX - int(t[400] - t[399])                                                          # one delta of 2^60 - 1: raw
    f[32] = t
    f[40] = I64_MIN + 1 + np.cumsum(rng.integers(1, 5, n)).astype(np.int64)                            # near INT64_MIN
    f[41] = (I64_MAX - np.cumsum(rng.integers(1, 5, n))[::-1]).astype(np.int64)                       # near INT64_MAX, INT64_MAX - 1 last
    f[42] = np.array([I64_MIN + 1, 0, I64_MAX - 1], np.int64)
    f[43] = I64_MIN + np.arange(n, dtype=np.int64) * 3      # a new series' row at INT64_MIN is at or before its last time: late
    return {sid: np.asarray(t, np.int64) for sid, t in f.items()}


def test_time_forms_through_a_flush():
    tf = _time_forms()
    rng = np.random.default_rng(37)
    assert (np.diff(tf[32]) == S8B_MAX).sum() == 1 and (np.diff(tf[31]) == S8B_MAX - 1).sum() == 1
    batch = {}
    for sid, t in tf.items():
        batch[sid] = _series(t, _cols(rng, t.size, ("fv", "iv"), 0.05))
    batch = _shuffle_and_repeat(rng, batch, 2)
    sh = Shard.open_rows(batch)
    files = fm.files(batch)
    tw = Shard.open_files(_descs(files))
    _twin_check(sh, tw, files)
    # the forms the cases exist for, from the flushed shard's own time pages
    ex = sh.export()
    nc = ex["col_types"].size
    forms = {}
    for u, sid in enumerate(ex["sids"].tolist()):
        for g in range(int(ex["series_seg_begin"][u]), int(ex["series_seg_begin"][u + 1])):
            p = ex["data"][int(ex["page_off"][nc][g]):int(ex["page_off"][nc][g]) + int(ex["page_len"][nc][g])]
            c = pf.time_codec(p)
            forms.setdefault(sid, set()).add((c, pf.time_s8b(p)[0]) if c == "t_s8b" else c)
    assert "t_const" in forms[1] and ("t_s8b", 1) in forms[2] and ("t_s8b", 1000) in forms[4] and ("t_s8b", 10**6) in forms[5]
    for k in (2, 3, 4, 5, 7, 8):
        assert ("t_s8b", 10**k) in forms[10 + k], (k, forms[10 + k])
    assert "t_raw" in forms[30] and "t_raw" in forms[32] and ("t_s8b", 1) in forms[31] and "t_raw" not in forms[31]
    # queries over bounded ranges of the regular series (the others span windows the query refuses or bins in the billions)
    sub = {sid: s for sid, s in _model(files).items() if sid < 30}
    one = Shard.open_files([(_file_desc(sub), False)])
    lo, hi = T0, T0 + 3000 * SEC
    for calls in ([("sum", 0), ("count", 0), ("max", 0)], [("min", 1), ("sum", 1), ("last", 1)]):
        for flags in (L.Q_STRICT_ORDER, L.Q_STRICT_ORDER | L.Q_NO_FUSED):
            qa = AggQuery(sh, calls, 60 * SEC, lo, hi, flags=flags, group="series").run()
            qb = AggQuery(one, calls, 60 * SEC, lo, hi, flags=flags, group="series").run()
            da, db = qa.dense_host(), qb.dense_host()
            na = qa.dense_host()["n_buckets"]
            # the flushed shard holds more series: compare the rows of the series both hold
            ia = [ex["sids"].tolist().index(s) for s in sorted(sub)]
            for ca, cb in zip(da["cols"], db["cols"]):
                va = np.concatenate([ca["values"][i * na:(i + 1) * na] for i in ia]).view(np.uint64)
                ka = np.concatenate([ca["valid"][i * na:(i + 1) * na] for i in ia])
                assert np.array_equal(ka, cb["valid"]) and np.array_equal(va[ka.astype(bool)], cb["values"].view(np.uint64)[ka.astype(bool)])
            qa.close(); qb.close()
    one.close(); sh.close(); tw.close()


def test_value_edges_through_flushes():
    """one time repeated (one row survives, each column its last non-null copy), ints at the limits and with zig-zag deltas past
    2^60 (raw pages), +Inf and -Inf without NaN in one segment (the raw page), a column null throughout the late part"""
    rng = np.random.default_rng(41)
    n = 2500
    t = T0 + np.arange(n, dtype=np.int64) * SEC
    iv = rng.integers(I64_MIN, I64_MAX, n, dtype=np.int64, endpoint=True)
    iv[[0, 1, 999, 1000, 1001, 2499]] = [I64_MIN, I64_MAX, I64_MIN, I64_MAX, 0, I64_MIN]
    fv = rng.standard_normal(n) * 100 + rng.random(n) * 1e-7
    fv[[3, 500]] = [np.inf, -np.inf]              # one segment: +Inf and -Inf, no NaN
    fv[[1200, 2100]] = [-np.inf, -np.inf]
    base = {5: _series(t, {"fv": (L.TYPE_FLOAT, fv, np.ones(n, bool)), "iv": (L.TYPE_INT, iv, rng.random(n) > 0.05),
                           "bv": (L.TYPE_BOOL, (rng.random(n) < 0.5).astype(np.uint8), np.ones(n, bool))}),
            6: _series(t, _cols(rng, n, ("fv", "iv", "bv"), 0.0))}
    tw = _twins_of_rows(base)
    assert "raw" in {pf.codec_of(L.TYPE_INT, p) for p in _column_pages(tw.sh, 5, 2)}      # columns bv, fv, iv
    assert pf.codec_of(L.TYPE_FLOAT, _column_pages(tw.sh, 5, 1)[0]) == "raw"
    # one time 40 times over, every column null in some copies; a wrapping int walk; late rows without bool values
    k = 40
    tt = np.full(k, T0 + (n + 10) * SEC)
    rep = {5: _series(tt, {"fv": (L.TYPE_FLOAT, rng.standard_normal(k), rng.random(k) < 0.3),
                           "iv": (L.TYPE_INT, rng.integers(I64_MIN, I64_MAX, k, dtype=np.int64), rng.random(k) < 0.3),
                           "bv": (L.TYPE_BOOL, (rng.random(k) < 0.5).astype(np.uint8), rng.random(k) < 0.3)})}
    m = 1500
    tl = np.concatenate([T0 + (n + 20 + np.arange(m, dtype=np.int64)) * SEC, T0 + np.arange(0, n, 5, dtype=np.int64) * SEC + SEC // 2])
    wrap = (I64_MAX - 3000 + np.arange(tl.size, dtype=np.int64).astype(object) * 7)
    wrap = np.array([int(x) & ((1 << 64) - 1) for x in wrap], np.uint64).view(np.int64)
    late_part = tl > t[-1]
    rep[6] = _series(tl, {"fv": (L.TYPE_FLOAT, rng.standard_normal(tl.size), np.ones(tl.size, bool)),
                          "iv": (L.TYPE_INT, wrap, np.ones(tl.size, bool)),
                          "bv": (L.TYPE_BOOL, np.ones(tl.size, np.uint8), late_part)})   # null throughout the out-of-order part
    info = tw.flush(rep, paths=False)
    assert info["rows_replaced"] == k - 1
    model = _model(tw.files)
    last = model[5]["times"].size - 1
    for name in ("fv", "iv", "bv"):
        _ty, v, ok = rep[5]["cols"][name]
        assert model[5]["cols"][name][2][last] == ok.any()
        if ok.any():
            assert model[5]["cols"][name][1][last] == v[np.flatnonzero(ok)[-1]]
    ooo = [f for f, o in tw.files if o][-1]
    assert "bv" not in ooo[6]["cols"]                # the late part of series 6 has no bool column
    tw.close()


def test_an_all_null_column_is_dropped_when_every_row_is_on_one_side():
    """A column null in every row of a series' part has no page there.  When the rows straddle the series' last time this is the
    reference's rule (SplitRecordByTime, engine/mutable/ts_table.go:276-286); when every row falls on one side the reference hands
    the record on unchanged (:243-248) and writes all-null pages, which the flush does not (DESIGN.md "Deviations").  A column
    null in every row of every flushed series is not a column of the shard."""
    rng = np.random.default_rng(43)
    n = 1200
    base = {sid: _series(T0 + np.arange(n, dtype=np.int64) * SEC, _cols(rng, n, ("fv", "iv"), 0.0)) for sid in (1, 2, 3, 4)}
    tw = _Twins([(base, False)])

    def with_null_bool(sid, t):
        c = _cols(rng, t.size, ("fv", "iv"), 0.1)
        c["bv"] = (L.TYPE_BOOL, np.zeros(t.size, np.uint8), np.zeros(t.size, bool))
        return _series(t, c)
    batch = {1: with_null_bool(1, T0 + (n + np.arange(1100, dtype=np.int64)) * SEC),          # every row after: ordered file
             2: with_null_bool(2, T0 + np.arange(0, n, 3, dtype=np.int64) * SEC + SEC // 2),   # every row before: out-of-order
             3: with_null_bool(3, T0 + (n - 50 + np.arange(100, dtype=np.int64)) * SEC),       # both sides: dropped
             9: with_null_bool(9, T0 + np.arange(10, dtype=np.int64) * SEC)}                  # a new sid: ordered file
    new = fm.files(batch, fm.last_times(tw.tw.export()))
    (fo, oo), (fx, ox) = new
    assert not oo and ox
    assert all("bv" not in f[sid]["cols"] for f in (fo, fx) for sid in f)
    tw.flush(batch, paths=False)
    assert tw.sh.export()["col_types"].tolist() == [L.TYPE_FLOAT, L.TYPE_INT]
    # a valid bool row in one series makes the column; the all-null series still get no bool page
    batch = {1: with_null_bool(1, T0 + (n + 1100 + np.arange(30, dtype=np.int64)) * SEC),
             4: with_null_bool(4, T0 + (n + np.arange(30, dtype=np.int64)) * SEC)}
    batch[4]["cols"]["bv"][2][7] = True
    tw.flush(batch, paths=False)
    assert tw.sh.export()["col_types"].tolist() == [L.TYPE_BOOL, L.TYPE_FLOAT, L.TYPE_INT]
    assert not _column_pages(tw.sh, 1, 0) and not _column_pages(tw.sh, 9, 0)
    pages = _column_pages(tw.sh, 4, 0)
    assert len(pages) == 1 and int(pages[0][0]) == L.TYPE_BOOL  # a bitmap page: one value in 30 rows
    tw.close()


# ---------------------------------------------------------------- histories
def _flush_step(sh, tw, files, batch):
    """one flush in a history: the rows into sh, the model's files into the twin, both checked"""
    step = fm.files(batch, fm.last_times(sh.export()))
    b = dict(step=step, n_rows=sh.info()["n_rows"])
    info = sh.append_rows(batch)
    tw.append_files(_descs(step))
    files += step
    _same_directory_and_pages(sh, tw)
    assert sh.info() == tw.info()
    _step_check(sh, files, b)
    return info


def _compact_both(sh, tw, files, R):
    b = dict(want=cm.expected(sh.export(), R), merge_info=sh.merge_info())
    b["info"] = sh.compact(R)
    tw.compact(R)
    _step_check(sh, files, b)
    _same_directory_and_pages(sh, tw)


def test_history_rows_compactions_and_files():
    """open_rows -> compact R = 7 -> late rows into the 7-row segments and across the last time -> a new column -> compact
    R = 1000 -> an out-of-order file -> a flush"""
    rng = np.random.default_rng(201)
    sids = [2, 4, 6]
    b0 = _shuffle_and_repeat(rng, {sid: _series(T0 + np.arange(300, dtype=np.int64) * SEC, _cols(rng, 300, ("fv", "iv"), 0.05)) for sid in sids}, 2)
    sh = Shard.open_rows(b0)
    files = fm.files(b0)
    tw = Shard.open_files(_descs(files))
    _twin_check(sh, tw, files)
    _step_check(sh, files)
    _compact_both(sh, tw, files, 7)
    late = {}
    for sid in sids[:2]:
        t = np.unique(np.concatenate([T0 + rng.integers(0, 300, 40) * SEC + SEC // 2, T0 + rng.integers(0, 300, 10) * SEC,
                                      T0 + (300 + np.arange(20, dtype=np.int64)) * SEC]))
        late[sid] = _series(t, _cols(rng, t.size, ("fv", "iv"), 0.2))
    _flush_step(sh, tw, files, _shuffle_and_repeat(rng, late, 3))
    new_col = {sid: _series(T0 + (330 + np.arange(50, dtype=np.int64)) * SEC, _cols(rng, 50, ("fv", "iv", "bv"), 0.1)) for sid in sids}
    for s_ in new_col.values():
        s_["cols"]["gv"] = (L.TYPE_FLOAT, rng.normal(0, 5, 50), rng.random(50) > 0.1)
    _flush_step(sh, tw, files, new_col)
    _compact_both(sh, tw, files, 1000)
    ooo = {sid: _series(np.unique(T0 + rng.integers(-30, 380, 60) * SEC + SEC // 4), None) for sid in sids[1:]}
    for s_ in ooo.values():
        s_["cols"] = _cols(rng, s_["times"].size, ("fv", "iv"), 0.1)
    step = [(ooo, True)]
    b = dict(step=step, n_rows=sh.info()["n_rows"])
    sh.append_files(_descs(step)); tw.append_files(_descs(step)); files += step
    _step_check(sh, files, b)
    _flush_step(sh, tw, files, _shuffle_and_repeat(rng, {sid: _series(T0 + (200 + np.arange(400, dtype=np.int64)) * SEC, _cols(rng, 400, ("fv", "iv", "bv"), 0.1))
                                                          for sid in sids + [5]}, 2))
    sh.close(); tw.close()


def test_rows_onto_a_written_and_reopened_file():
    rng = np.random.default_rng(202)
    sids = [10, 20, 30]
    first = {sid: _series(T0 + np.arange(1800, dtype=np.int64) * SEC, _cols(rng, 1800, ("fv", "iv", "bv"), 0.05)) for sid in sids}
    src = Shard.open_rows(first)
    img = write_tssp(src, "m")
    src.close()
    files = [(first, False)]
    sh, tw = Shard.open_files([(img, False)]), Shard.open_files([(img, False)])
    _step_check(sh, files)
    batch = {sid: _series(np.concatenate([T0 + (1800 + np.arange(700, dtype=np.int64)) * SEC, T0 + np.arange(3, 1800, 11, dtype=np.int64) * SEC + 7]),
                          None) for sid in (10, 25, 30)}
    for s_ in batch.values():
        s_["cols"] = _cols(rng, s_["times"].size, ("fv", "iv"), 0.1)
    batch[25]["times"] = batch[25]["times"] + 3 * SEC  # a new sid between the file's
    _flush_step(sh, tw, files, _shuffle_and_repeat(rng, batch, 3))
    _flush_step(sh, tw, files, {sid: _series(T0 + (2600 + np.arange(900, dtype=np.int64)) * SEC, _cols(rng, 900, ("fv", "iv"), 0.0)) for sid in sids})
    sh.close(); tw.close()


def test_rows_onto_snappy_pages():
    """few-decimal floats: the reference's files hold Snappy float pages, which the shard transcodes as they come in; late rows
    then merge into those segments, new rows follow them"""
    rng = np.random.default_rng(203)
    n = 2000
    t = T0 + np.arange(n, dtype=np.int64) * SEC
    snappy = {sid: _series(t, {"fv": (L.TYPE_FLOAT, np.round(rng.normal(100, 20, n), 2), np.ones(n, bool)),
                               "iv": (L.TYPE_INT, np.arange(n) * sid, np.ones(n, bool))}) for sid in (1, 2)}
    files = [(snappy, False)]
    d = _file_desc(snappy)
    assert any(pf.codec_of(L.TYPE_FLOAT, p) == "snappy" for p in _pages_of_desc(snappy))
    sh, tw = Shard.open_files([(d, False)]), Shard.open_files([(_file_desc(snappy), False)])
    _step_check(sh, files)
    late = {1: _series(np.concatenate([T0 + np.arange(5, 1500, 13, dtype=np.int64) * SEC + SEC // 2, t[-1] + SEC * np.arange(1, 300)]), None)}
    late[1]["cols"] = {"fv": (L.TYPE_FLOAT, rng.normal(100, 20, late[1]["times"].size), np.ones(late[1]["times"].size, bool)),
                       "iv": (L.TYPE_INT, rng.integers(-5, 5, late[1]["times"].size), np.ones(late[1]["times"].size, bool))}
    _flush_step(sh, tw, files, _shuffle_and_repeat(rng, late, 2))
    sh.close(); tw.close()


def _pages_of_desc(series):
    _names, _types, segs = fm.file_pages(series)
    return [p for _sid, ss in segs for _lo, _hi, pages, _tp in ss for nm, p in pages.items() if nm == "fv"]


def test_downsample_after_flushes():
    """og_downsample_shard of a shard built by flushes with late rows against that of the same rows opened as one file: the same
    sids, rows and cells bit for bit, float sums within 1e-12 relative (the two shards cut their rows into different segments)"""
    rng = np.random.default_rng(204)
    sids = [3, 9, 27]
    b0 = {sid: _series(T0 + np.arange(2000, dtype=np.int64) * SEC, _cols(rng, 2000, ("fv", "iv"), 0.05)) for sid in sids}
    tw = _twins_of_rows(b0)
    late = {sid: _series(np.unique(T0 + rng.integers(-100, 2300, 300) * SEC + SEC // 2), None) for sid in sids[:2]}
    for s_ in late.values():
        s_["cols"] = _cols(rng, s_["times"].size, ("fv", "iv"), 0.2)
    tw.flush(_shuffle_and_repeat(rng, late, 2), paths=False)
    tw.flush({sid: _series(T0 + (2400 + np.arange(700, dtype=np.int64)) * SEC, _cols(rng, 700, ("fv", "iv"), 0.0)) for sid in sids}, paths=False)
    model = _model(tw.files)
    one = Shard.open_files([(_file_desc(model), False)])
    tmin = min(int(s["times"][0]) for s in model.values())
    tmax = max(int(s["times"][-1]) for s in model.values())
    ops = {L.TYPE_FLOAT: ["sum", "count", "min", "max", "first", "last"], L.TYPE_INT: ["sum", "min", "last"]}
    da, db = tw.sh.downsample_shard(IV, tmin, tmax, ops), one.downsample_shard(IV, tmin, tmax, ops)
    xa, xb = da.open(), db.open()
    ea, eb = xa.export(), xb.export()
    assert np.array_equal(ea["sids"], eb["sids"]) and ea["sids"].tolist() == sorted(model)
    names = [c[0] for c in da.columns()[0]]
    for u in range(ea["sids"].size):
        ra = [xa.decode_segment(g) for g in range(int(ea["series_seg_begin"][u]), int(ea["series_seg_begin"][u + 1]))]
        rb = [xb.decode_segment(g) for g in range(int(eb["series_seg_begin"][u]), int(eb["series_seg_begin"][u + 1]))]
        assert np.array_equal(np.concatenate([r["times"] for r in ra]), np.concatenate([r["times"] for r in rb])), u
        for c, name in enumerate(names):
            va, vb = np.concatenate([r["cols"][c]["valid"] for r in ra]), np.concatenate([r["cols"][c]["valid"] for r in rb])
            xa_, xb_ = np.concatenate([r["cols"][c]["values"] for r in ra]), np.concatenate([r["cols"][c]["values"] for r in rb])
            assert np.array_equal(va, vb), (u, name)
            if name == "sum_fv":
                assert np.all(np.abs(xa_ - xb_) <= 1e-12 * np.maximum(1.0, np.abs(xb_))), (u, name)
            else:
                assert np.array_equal(xa_.view(np.uint8), xb_.view(np.uint8)), (u, name)
    xa.close(); xb.close(); da.close(); db.close(); one.close()
    _step_check(tw.sh, tw.files)
    tw.close()


def test_a_long_flush_compact_query_loop_leaves_no_device_memory_behind():
    """thirty steps: flushes of new and late rows (repeated and shuffled), compactions at changing R and a query on every step;
    the data region holds only live pages after every step, rows against the model every few steps, pages against the twin at
    the end, and closing the shards returns every buffer"""
    rng = np.random.default_rng(205)
    sids = [1, 2, 3, 4, 5]
    Rs = [7, 1000, 50, 999, 13, 1000, 300, 1]
    with _NoLeak():
        b0 = {sid: _series(T0 + np.arange(200, dtype=np.int64) * SEC, _cols(rng, 200, ("fv", "iv", "bv"), 0.05)) for sid in sids}
        sh = Shard.open_rows(b0)
        files = fm.files(b0)
        tw = Shard.open_files(_descs(files))
        for k in range(30):
            model = _model(files)
            if k % 4 == 3:
                R = Rs[(k // 4) % len(Rs)]
                sh.compact(R); tw.compact(R)
            else:
                batch = {}
                for sid in sids[k % 2::2] + ([6 + k] if k % 5 == 0 else []):
                    last = int(model[sid]["times"][-1]) if sid in model else T0
                    t = last + SEC * np.arange(1, 2 + int(rng.integers(0, 40)), dtype=np.int64)
                    if sid in model and k % 3:
                        t = np.concatenate([t, np.unique(last - rng.integers(0, 150, 15) * SEC - SEC // 3)])
                    batch[sid] = _series(t, _cols(rng, t.size, ("fv", "iv", "bv"), 0.1))
                batch = _shuffle_and_repeat(rng, batch, 3)
                step = fm.files(batch, fm.last_times(sh.export()))
                sh.append_rows(batch); tw.append_files(_descs(step)); files += step
            assert _data_excess(sh) == 0, k
            q = AggQuery(sh, [("count", 1), ("sum", 2)], IV, T0, T0 + 5000 * SEC, flags=L.Q_STRICT_ORDER).run()
            q.dense_host(); q.close()
            if k % 7 == 6:
                _check_rows(sh, _model(files))
        _twin_check(sh, tw, files)
        _step_check(sh, files)
        sh.close(); tw.close()
