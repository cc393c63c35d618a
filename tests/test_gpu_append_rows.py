"""og_shard_append_rows / og_shard_open_rows: a memtable flush sorted, split and encoded on the device.

Every flush is checked three ways: against og_shard_append_files of the two files tests/flush_model.py writes for the same rows on a
twin shard (directory, every page byte, og_shard_info and og_shard_merge_info), row by row against the merged model of every file
so far (test_gpu_out_of_order._model), and on every query path against the oracle's file-set read (test_gpu_append._all_paths)."""

import numpy as np
import pytest

import flush_model as fm
from opengemini_b200 import AggQuery, Shard, write_tssp
from opengemini_b200 import _lib as L
from test_gpu_append import _all_paths, _cols, _dense_equal, _same_directory_and_pages, _snapshot, _unchanged
from test_gpu_device_memory import _NoLeak
from test_gpu_out_of_order import ALL6, SEC, T0, _check_rows, _model, _series
from test_gpu_threads import _answer, _run_threads

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module", autouse=True)
def _device():
    Shard.init(0)


def _descs(files):
    return [(fm.file_desc(f), ooo) for f, ooo in files]


def _same_merge_info(a, b):
    ma, mb = a.merge_info(), b.merge_info()
    ma.pop("merge_ms"); mb.pop("merge_ms")
    assert ma == mb


class _Twins:
    """a shard that takes rows and its twin that takes the model's files; `files` holds every file either holds so far"""

    def __init__(self, base_files):
        self.files = list(base_files)
        self.sh = Shard.open_files(_descs(base_files))
        self.tw = Shard.open_files(_descs(base_files))

    def flush(self, batch, paths=True):
        new = fm.files(batch, fm.last_times(self.tw.export()))
        info = self.sh.append_rows(batch)
        self.tw.append_files(_descs(new))
        self.files += new
        _same_directory_and_pages(self.sh, self.tw)
        assert self.sh.info() == self.tw.info()
        _same_merge_info(self.sh, self.tw)
        _check_rows(self.sh, _model(self.files))
        assert info["rows_in"] == sum(len(s["times"]) for s in batch.values())
        assert info["ordered_rows"] + info["out_of_order_rows"] + info["rows_replaced"] == info["rows_in"]
        assert info["out_of_order_rows"] == sum(s["times"].size for f, ooo in new if ooo for s in f.values())
        if paths:
            _all_paths(self.sh, self.files)
        return info

    def close(self):
        self.sh.close(); self.tw.close()


def _shuffle_and_repeat(rng, batch, max_rep=5):
    """times repeated 1-5x (later copies with fresh values and more nulls) and shuffled: the arrival order of a memtable"""
    out = {}
    for sid, s in batch.items():
        n = s["times"].size
        rep = rng.integers(1, max_rep + 1, n)
        idx = np.repeat(np.arange(n), rep)
        perm = rng.permutation(idx.size)
        idx = idx[perm]
        cols = {}
        for name, (t, v, ok) in s["cols"].items():
            vv = np.array(v)[idx]
            noise = rng.random(idx.size) < 0.5
            if t == L.TYPE_FLOAT:
                vv = np.where(noise, vv + rng.random(idx.size), vv)
            elif t == L.TYPE_INT:
                vv = np.where(noise, vv + rng.integers(1, 9, idx.size), vv)
            cols[name] = (t, vv.astype(np.asarray(v).dtype), np.asarray(ok)[idx] & (rng.random(idx.size) >= 0.3))
        out[sid] = _series(s["times"][idx], cols)
    return out


def _rows(rng, sids, t_lo, n, present=("fv", "iv", "bv"), null_p=0.05, step=1):
    t = T0 + (t_lo + np.arange(n, dtype=np.int64) * step) * SEC
    return {sid: _series(t, _cols(rng, n, present, null_p)) for sid in sids}


# ---------------------------------------------------------------- flushes against the model's files
@pytest.mark.parametrize("batch_rows", [None, "1500"])
def test_flushes_equal_appending_the_model_files(batch_rows, monkeypatch):
    if batch_rows:
        monkeypatch.setenv("OGPU_MERGE_BATCH_ROWS", batch_rows)  # many batches: the same bytes
    rng = np.random.default_rng(5)
    sids = [20, 30, 40, 50]
    tw = _Twins([(_rows(rng, sids, 0, 2600), False)])
    # ordered only: sids that sort first and into the middle, a series without the bool column, unsorted and repeated times
    b = _rows(rng, [10, 25, 30, 40], 2600, 1300)
    b[25]["cols"].pop("bv")
    tw.flush(_shuffle_and_repeat(rng, b))
    # every row at or before the series' last time; one row at exactly the last time
    late = {}
    for sid in (20, 30):
        t = np.unique(T0 + rng.integers(-50, 2600, 300) * SEC + np.where(rng.random(300) < 0.3, SEC // 2, 0))
        late[sid] = _series(t, _cols(rng, t.size, ("fv", "iv"), 0.2))
    late[30]["times"][-1] = T0 + 3899 * SEC  # series 30's last time (2600 + 1299)
    late[30]["times"].sort()
    tw.flush(_shuffle_and_repeat(rng, late, 3))
    # a mix: new rows after the last time and late rows, a new column that sorts last, a new sid
    mix = _rows(rng, [20, 30, 40, 60], 3900, 900, null_p=0.4)
    for sid in (20, 60):
        tl = T0 + rng.integers(0, 3900, 80) * SEC + SEC // 3
        mix[sid] = _series(np.concatenate([mix[sid]["times"], tl]),
                           {n: (t, np.concatenate([v, np.asarray(v)[:80]]), np.concatenate([ok, np.ones(80, bool)])) for n, (t, v, ok) in mix[sid]["cols"].items()})
    for s in mix.values():
        s["cols"]["zz"] = (L.TYPE_INT, np.arange(s["times"].size), np.ones(s["times"].size, bool))
    tw.flush(_shuffle_and_repeat(rng, mix, 2))
    tw.close()


@pytest.mark.parametrize("typ", [L.TYPE_INT, L.TYPE_FLOAT, L.TYPE_BOOL])
def test_null_ratios_and_bitmap_offsets(typ):
    rng = np.random.default_rng(typ)
    n = 1700
    sids = [1, 2, 3, 4]
    base = _rows(rng, sids, 0, 1200)
    tw = _Twins([(base, False)])
    t = T0 + (1200 + np.arange(n, dtype=np.int64)) * SEC
    t_late = T0 + np.arange(0, 1200, 4, dtype=np.int64) * SEC + SEC // 2
    tt = np.concatenate([t, t_late])
    series, batch = [], {}
    for k, (sid, null_p, off, bitmap) in enumerate([(1, 0.0, 0, False), (2, 0.05, 3, True), (3, 0.4, 13, True), (4, 1.0, 0, True)]):
        valid = rng.random(tt.size) >= null_p
        v = {L.TYPE_INT: rng.integers(-(1 << 40), 1 << 40, tt.size), L.TYPE_FLOAT: np.round(rng.normal(0, 50, tt.size), 4) + rng.random(tt.size) * 1e-7,
             L.TYPE_BOOL: (rng.random(tt.size) < 0.5).astype(np.uint8)}[typ]
        fv = (L.TYPE_FLOAT, rng.normal(100, 20, tt.size), np.ones(tt.size, bool))
        iv = (L.TYPE_INT, rng.integers(-9, 9, tt.size).cumsum(), rng.random(tt.size) >= 0.1)
        batch[sid] = _series(tt, {"fv": fv, "iv": iv, "x": (typ, v, valid)})
        series.append((sid, tt, [Shard.colval(*fv), Shard.colval(*iv), Shard.colval(typ, v, valid, bitmap_offset=off, bitmap=bitmap)]))
    d = Shard.rows_desc([("fv", L.TYPE_FLOAT), ("iv", L.TYPE_INT), ("x", typ)], series)
    new = fm.files(batch, fm.last_times(tw.tw.export()))
    tw.sh.append_rows(d)
    tw.tw.append_files(_descs(new))
    tw.files += new
    _same_directory_and_pages(tw.sh, tw.tw)
    assert tw.sh.info() == tw.tw.info()
    _same_merge_info(tw.sh, tw.tw)
    _check_rows(tw.sh, _model(tw.files))
    _all_paths(tw.sh, tw.files)
    tw.close()


def _same_as_model(sh, ref, files):
    _same_directory_and_pages(sh, ref)
    assert sh.info() == ref.info()
    _same_merge_info(sh, ref)
    _check_rows(sh, _model(files))


def test_special_floats():
    n = 1500
    t = T0 + np.arange(n, dtype=np.int64) * SEC
    rng = np.random.default_rng(3)
    v = np.round(rng.normal(0, 9, n), 3) + rng.random(n) * 1e-6
    v[[5, 10, 700]] = [np.nan, np.inf, -np.inf]  # one segment holds NaN, +Inf and -Inf: the raw page
    v[1200:1210] = [0.0, -0.0] * 5              # signed zeros keep their bits
    w = np.round(rng.normal(0, 9, n), 3) + rng.random(n) * 1e-6
    w[[3, 400]] = np.nan                         # NaN alone in a segment: the raw page too
    ok = np.ones(n, bool)
    batch = {9: _series(t, {"fv": (L.TYPE_FLOAT, v, ok)}), 11: _series(t, {"fv": (L.TYPE_FLOAT, w, ok)})}
    sh = Shard.open_rows(batch)
    files = fm.files(batch)
    ref = Shard.open_files(_descs(files))
    _same_as_model(sh, ref, files)
    # a second flush: late rows with NaN and infinities landing on the first segment, and new rows after it
    tl = T0 + np.arange(0, 900, 9, dtype=np.int64) * SEC + SEC // 2
    x = rng.normal(0, 9, tl.size) + rng.random(tl.size) * 1e-6
    x[[1, 7, 20]] = [np.nan, np.inf, -np.inf]
    u = v[::-1].copy()
    nb = {9: _series(np.concatenate([t + n * SEC, tl]), {"fv": (L.TYPE_FLOAT, np.concatenate([u, x]), np.ones(n + tl.size, bool))})}
    new = fm.files(nb, fm.last_times(ref.export()))
    assert [o for _f, o in new] == [False, True]
    sh.append_rows(nb)
    ref.append_files(_descs(new))
    files += new
    _same_as_model(sh, ref, files)
    sh.close(); ref.close()


def _pool(attr, value=None):
    """the default memory pool's attribute `attr` (CU_MEMPOOL_ATTR_*), set to `value` first when given"""
    import ctypes as C
    L.check(L.lib().og_release_cached_memory(), "og_release_cached_memory")
    cu = C.CDLL("libcuda.so.1")
    dev, pool, v = C.c_int(), C.c_void_p(), C.c_uint64(0 if value is None else value)
    assert cu.cuInit(0) == 0 and cu.cuDeviceGet(C.byref(dev), 0) == 0 and cu.cuDeviceGetDefaultMemPool(C.byref(pool), dev) == 0
    if value is not None:
        assert cu.cuMemPoolSetAttribute(pool, attr, C.byref(v)) == 0
    assert cu.cuMemPoolGetAttribute(pool, attr, C.byref(v)) == 0
    return v.value


USED_CURRENT, USED_HIGH = 7, 8  # CU_MEMPOOL_ATTR_USED_MEM_CURRENT / _HIGH


def test_many_short_series_stay_inside_the_batch_budget(monkeypatch):
    """20 000 series of 1-3 rows, some late: every series costs whole output segments, so the batch budget must charge them.
    Under a budget of 60 000 row-equivalents a batch holds a few dozen series, and the pool's peak stays far below the
    ~40 000 segments' worth (several GB) one batch of every series would ask for."""
    rng = np.random.default_rng(41)
    n_ser = 20000
    sids = list(range(1, 2 * n_ser, 2))
    base = {sid: _series(T0 + np.arange(2, dtype=np.int64) * 10 * SEC, _cols(rng, 2, ("fv", "iv"), 0.0)) for sid in sids[::2]}
    tw = _Twins([(base, False)])
    batch = {}
    for sid in sids:
        k = int(rng.integers(1, 4))
        t = T0 + (20 + np.arange(k, dtype=np.int64)) * SEC
        if sid in base and rng.random() < 0.5:
            t[0] = T0 + 5 * SEC                  # a late row between the base's two
        batch[sid] = _series(t, _cols(rng, k, ("fv", "iv", "bv"), 0.2))
    monkeypatch.setenv("OGPU_MERGE_BATCH_ROWS", "60000")
    before = _pool(USED_CURRENT)
    _pool(USED_HIGH, 0)
    info = tw.flush(batch, paths=False)
    peak = _pool(USED_HIGH) - before
    assert info["out_of_order_rows"] > 1000
    assert peak < 1 << 30, peak
    tw.close()


def test_a_long_series_spreads_over_expand_chunks():
    """one series of 50 000 rows (expand tasks of 8192 rows: the dense index of each chunk starts where the last one ended),
    nulls behind a bitmap that starts at bit 5, and late rows"""
    rng = np.random.default_rng(43)
    n = 50000
    tw = _Twins([(_rows(rng, [7], 0, 3000), False)])
    t = np.concatenate([T0 + (3000 + np.arange(n, dtype=np.int64)) * SEC, T0 + np.arange(0, 3000, 7, dtype=np.int64) * SEC + SEC // 2])
    perm = rng.permutation(t.size)
    cols = {"fv": (L.TYPE_FLOAT, rng.normal(100, 20, t.size)[perm], (rng.random(t.size) >= 0.4)),
            "iv": (L.TYPE_INT, rng.integers(-9, 9, t.size).cumsum(), rng.random(t.size) >= 0.05)}
    batch = {7: _series(t[perm], cols)}
    series = [(7, t[perm], [Shard.colval(*cols["fv"], bitmap_offset=5), Shard.colval(*cols["iv"], bitmap_offset=13)])]
    new = fm.files(batch, fm.last_times(tw.tw.export()))
    tw.sh.append_rows(Shard.rows_desc([("fv", L.TYPE_FLOAT), ("iv", L.TYPE_INT)], series))
    tw.tw.append_files(_descs(new))
    tw.files += new
    _same_as_model(tw.sh, tw.tw, tw.files)
    _all_paths(tw.sh, tw.files)
    tw.close()


@pytest.mark.parametrize("n", [1, 999, 1000, 1001, 2500])
def test_part_sizes(n):
    rng = np.random.default_rng(n)
    tw = _Twins([(_rows(rng, [5, 6], 0, 3000, step=2), False)])
    late = {5: _series(T0 + (np.arange(n, dtype=np.int64) * 2 + 1) * SEC, _cols(rng, n, ("fv", "iv"), 0.1))}
    new = {6: _series(T0 + (6000 + np.arange(n, dtype=np.int64)) * SEC, _cols(rng, n, ("fv", "iv", "bv"), 0.1))}
    tw.flush(_shuffle_and_repeat(rng, {**late, **new}, 2), paths=n >= 1000)
    tw.close()


def test_open_rows_equals_opening_the_model_file():
    rng = np.random.default_rng(11)
    batch = _shuffle_and_repeat(rng, _rows(rng, [3, 1, 2], 0, 2100))
    sh = Shard.open_rows(batch)
    (f, ooo), = fm.files(batch)
    assert not ooo
    ref = Shard.open_files([(fm.file_desc(f), False)])
    _same_directory_and_pages(sh, ref)
    assert sh.info() == ref.info()
    _same_merge_info(sh, ref)
    assert sh.rows_info["rows_replaced"] == sum(len(s["times"]) for s in batch.values()) - sum(s["times"].size for s in f.values())
    _check_rows(sh, _model([(f, False)]))
    sh.close(); ref.close()


def test_a_regular_flush_into_a_synth_shard_keeps_the_folded_path():
    cols = [(L.TYPE_FLOAT, L.SYNTH_F_HI, 0), (L.TYPE_INT, L.SYNTH_INT_WALK, 0)]
    base = Shard.synth(300, 2000, cols, t0=T0, dt=SEC, seed=3)
    twin = Shard.synth(300, 2000, cols, t0=T0, dt=SEC, seed=3)
    sids = base.export()["sids"].tolist()
    rng = np.random.default_rng(4)
    t = T0 + (2000 + np.arange(1000, dtype=np.int64)) * SEC
    batch = {sid: _series(t, {"f0": (L.TYPE_FLOAT, rng.normal(50, 10, 1000), np.ones(1000, bool)),
                              "f1": (L.TYPE_INT, rng.integers(-5, 5, 1000).cumsum(), np.ones(1000, bool))}) for sid in sids}
    batch = _shuffle_and_repeat(rng, batch, 2)
    base.append_rows(batch)
    twin.append_files(_descs(fm.files(batch, fm.last_times(twin.export()))))
    _same_directory_and_pages(base, twin)
    assert base.info() == twin.info()
    for calls in ([("sum", 0), ("count", 0), ("max", 0)], [(f, 0) for f in ALL6]):
        assert _dense_equal(base, twin, calls, 60 * SEC, T0, T0 + 2999 * SEC) == 3
        _dense_equal(base, twin, calls, 60 * SEC, T0, T0 + 2999 * SEC, flags=L.Q_STRICT_ORDER)
    base.close(); twin.close()


# ---------------------------------------------------------------- a history, refusals, memory, threads
def test_rows_compact_late_rows_write_and_reopen():
    rng = np.random.default_rng(17)
    sids = [4, 8, 15]
    b0 = _rows(rng, sids, 0, 700, ("fv", "iv"))
    sh = Shard.open_rows(b0)
    files = fm.files(b0)
    for k in range(3):                           # small flushes, then compaction
        b = _rows(rng, sids, 700 + 300 * k, 300, ("fv", "iv"))
        files += fm.files(b, fm.last_times(sh.export()))
        sh.append_rows(b)
    sh.compact()
    late = {sid: _series(np.sort(T0 + rng.choice(1599, 120, replace=False) * SEC + SEC // 4), _cols(rng, 120, ("fv", "iv"), 0.2)) for sid in sids[:2]}
    late = _shuffle_and_repeat(rng, late, 2)
    files += fm.files(late, fm.last_times(sh.export()))
    sh.append_rows(late)
    assert files[-1][1]
    model = _model(files)
    _check_rows(sh, model)
    re = Shard.open_tssp(write_tssp(sh, "m"))
    _check_rows(re, model)
    re.close(); sh.close()


def test_refusals_leave_the_shard_as_it_was():
    rng = np.random.default_rng(23)
    n = 1200
    t = T0 + np.arange(n, dtype=np.int64) * SEC
    base = {sid: _series(t, {"a": (L.TYPE_FLOAT, rng.normal(0, 1, n), np.ones(n, bool)), "v": (L.TYPE_FLOAT, rng.normal(0, 1, n), np.ones(n, bool))})
            for sid in (1, 2)}
    sh = Shard.open_rows(base)
    snap = _snapshot(sh)  # column 1: "v"
    tn = t[-1] + SEC * np.arange(1, 11)
    good = Shard.colval(L.TYPE_FLOAT, np.arange(10.0), np.ones(10, bool))

    def refused(d, status, text=None):
        with pytest.raises(L.OgpuError) as ei:
            sh.append_rows(d)
        assert ei.value.status == status, str(ei.value)
        if text:
            assert text in str(ei.value), str(ei.value)
        _unchanged(sh, snap)

    refused(Shard.rows_desc([("s", 4)], [(2, tn, [None])]), L.OG_E_UNSUPPORTED, '"s"')
    refused(Shard.rows_desc([("v", L.TYPE_INT)], [(2, tn, [Shard.colval(L.TYPE_INT, np.arange(10), np.ones(10, bool))])]), L.OG_E_TYPE, '"v"')
    refused(Shard.rows_desc([("v", L.TYPE_FLOAT)], [(0, tn, [good])]), L.OG_E_INVAL, "sid 0")
    refused(Shard.rows_desc([("v", L.TYPE_FLOAT)], [(2, tn, [good]), (2, tn, [good])]), L.OG_E_INVAL, "twice")
    refused(Shard.rows_desc([("v", L.TYPE_FLOAT), ("v", L.TYPE_FLOAT)], [(2, tn, [good, good])]), L.OG_E_INVAL, "twice")
    refused(Shard.rows_desc([("v", L.TYPE_FLOAT)], [(2, tn, [dict(good, len=5)])]), L.OG_E_INVAL, "len")
    half = Shard.colval(L.TYPE_FLOAT, np.arange(10.0), np.arange(10) % 2 == 0)
    refused(Shard.rows_desc([("v", L.TYPE_FLOAT)], [(2, tn, [dict(half, nil_count=4, val=np.zeros(48, np.uint8))])]), L.OG_E_INVAL, "nil_count")
    refused(Shard.rows_desc([("v", L.TYPE_FLOAT)], [(2, tn, [dict(half, bitmap=None)])]), L.OG_E_INVAL, "nil_count")
    refused(Shard.rows_desc([("v", L.TYPE_FLOAT)], [(2, tn, [dict(half, val_bytes=48)])]), L.OG_E_INVAL, "val_bytes")
    refused(Shard.rows_desc([("v", L.TYPE_FLOAT)], [(2, tn, [good])], flags=1), L.OG_E_INVAL, "flags")
    q = AggQuery(sh, [("count", 0)], 0, T0, T0 + 2 * n * SEC)
    refused(Shard.rows_desc([("v", L.TYPE_FLOAT)], [(2, tn, [good])]), L.OG_E_STATE, "queries")
    q.close()
    sh.append_rows(Shard.rows_desc([("v", L.TYPE_FLOAT)], [(2, tn, [good])]))  # a valid flush after every refusal
    q = AggQuery(sh, [("count", 1)], 0, T0, T0 + 2 * n * SEC, group="series", flags=L.Q_STRICT_ORDER).run()
    assert q.dense_host()["cols"][0]["values"].tolist() == [n, n + 10]
    q.close(); sh.close()


def test_repeated_flushes_leave_no_device_memory_behind():
    rng = np.random.default_rng(29)
    with _NoLeak():
        sh = Shard.open_rows(_rows(rng, [1, 2, 3], 0, 1500))
        for k in range(4):
            b = _rows(rng, [1, 2, 3, 4], 1500 + 500 * k, 500)
            b[1] = _series(np.concatenate([b[1]["times"], T0 + np.arange(10, dtype=np.int64) * SEC + SEC // 2]),
                           {n: (t, np.concatenate([v, np.asarray(v)[:10]]), np.concatenate([ok, ok[:10]])) for n, (t, v, ok) in b[1]["cols"].items()})
            sh.append_rows(b)
        with pytest.raises(L.OgpuError):
            sh.append_rows(Shard.rows_desc([("fv", L.TYPE_INT)], [(1, np.array([T0 * 2]), [Shard.colval(L.TYPE_INT, [1], [True])])]))
        sh.close()


def test_a_query_created_during_a_flush_answers_as_before_or_after():
    cols = [(L.TYPE_FLOAT, L.SYNTH_F_HI, 0), (L.TYPE_FLOAT, L.SYNTH_F_LO, 0), (L.TYPE_INT, L.SYNTH_INT_WALK, 0)]
    sh = Shard.synth(16, 2000, cols, t0=T0, dt=SEC, seed=31)
    twin = Shard.synth(16, 2000, cols, t0=T0, dt=SEC, seed=31)
    rng = np.random.default_rng(31)
    t = T0 + (2000 + np.arange(700, dtype=np.int64)) * SEC
    batch = {int(sid): _series(t, {"f0": (L.TYPE_FLOAT, rng.normal(0, 1, 700), np.ones(700, bool))}) for sid in sh.export()["sids"]}
    tmax = T0 + 3000 * SEC
    calls, kw = [("sum", 0), ("count", 0), ("max", 0)], dict(group="series")
    before = _answer(sh, calls, kw, tmax)[:2]
    twin.append_rows(batch)
    after = _answer(twin, calls, kw, tmax)[:2]
    assert before != after

    def mutator():
        try:
            sh.append_rows(batch)
            return L.OG_OK
        except L.OgpuError as e:
            assert e.status == L.OG_E_STATE, str(e)
            return e.status

    status, got = _run_threads([mutator, lambda: _answer(sh, calls, kw, tmax)[:2]])
    if status == L.OG_E_STATE:
        sh.append_rows(batch)
    assert got == before or got == after
    assert _answer(sh, calls, kw, tmax)[:2] == after
    sh.close(); twin.close()
