"""Every aggregate, decode and write path on shards whose segments are not 1000 rows long.

openGemini's segment length is a setting (`max-rows-per-segment`), so a file may hold segments of any length, and a merge of a
longer-segment file leaves series that mix lengths.  The library has thresholds that depend on it: k_fused_cols (path 5) takes a
shard only if its longest segment has <= 1024 rows; the lane-interleaved copy takes segments of 2 .. 2^22 - 1 rows; a folding
warp accumulates at most OG_IL_WCAP (24) windows of a segment; the round watchdog of k_fused_il scales with the longest lane of a
group; descending materialisation takes segments of up to 65536 rows; the tile path sizes its tile by the longest segment.

Shards come from tests/segment_shards.py (the oracle's encoders over per-series rows cut at explicit lengths).  Every aggregate
names its path and asserts it from og_stats, then compares with oracle.scan: bitwise in strict order, float sums within SUM_RTOL
in the default order.  Re-cutting the same rows must not change any answer (checked against the numpy model, without the
oracle)."""
import numpy as np
import pytest
import torch

import oracle
import segment_shards as ss
from opengemini_b200 import AggQuery, ScanCursor, Shard, write_tssp
from opengemini_b200 import _lib as L
from test_gpu_parity import compare_dense

pytestmark = pytest.mark.gpu

T0, SEC = ss.T0, ss.SEC
ALL6 = ["count", "sum", "min", "max", "first", "last"]
SHORT = [1, 2, 3, 31, 32, 33, 999, 1000, 1001, 1023, 1024]
LONG = [2048, 4095, 4096, 8192, 65535, 65536, 65537]
KINDS = ["f_hi", "f_raw", "f_lo", "i_s8b", "i_const", "bool", "i_wide"]
NULLS = [0, 0, 0.1, 0.05, 0, 0.3, 0]  # bitmaps in f_lo, i_s8b and bool
TYPES = ss.types_of(KINDS)
FHI, FRAW, FLO, IS8B, ICONST, BOOL, IWIDE = range(len(KINDS))
FLAGS = {0: L.Q_STRICT_ORDER | L.Q_NO_FUSED, 1: L.Q_STRICT_ORDER | L.Q_NO_FAST, 2: L.Q_STRICT_ORDER, 3: 0, 4: L.Q_STRICT_ORDER,
         5: L.Q_STRICT_ORDER}


@pytest.fixture(scope="module", autouse=True)
def _device():
    Shard.init(0)


def _agg(sh, sd, calls, iv, tmin, tmax, path, monkeypatch, label, **kw):
    """Run the query the way `path` names, assert the path and compare with the oracle.  Path 3 runs twice (the second run of the
    same plan reuses its scratch); paths 4 and 5 also run in the default order for one tagset (float sums within SUM_RTOL)."""
    with monkeypatch.context() as m:
        if path == 4:
            m.setenv("OGPU_NO_COLS", "1")
        q = AggQuery(sh, calls, iv, tmin, tmax, flags=FLAGS[path], **kw).run()
        try:
            st = q.stats()
            assert st["path"] == path, f"{label}: path {st['path']}, wanted {path}"
            ref = oracle.scan(sd, q.desc, threads=1)
            compare_dense(q.dense_host(), ref, calls, len(calls) > 1, f"{label} [path {path}]", float_sum_exact=path != 3)
            if path == 3:
                q.run()
                compare_dense(q.dense_host(), ref, calls, len(calls) > 1, f"{label} [path 3, rerun]", float_sum_exact=False)
            else:
                assert st["rows_decoded"] == ref["rows_decoded"] and st["page_bytes"] == ref["page_bytes"], label
        finally:
            q.close()
        if path in (4, 5) and kw.get("group", "all") == "all":
            q = AggQuery(sh, calls, iv, tmin, tmax, **kw).run()
            try:
                assert q.stats()["path"] == path, label
                compare_dense(q.dense_host(), ref, calls, len(calls) > 1, f"{label} [path {path}, default order]", float_sum_exact=False)
            finally:
                q.close()
    return st


def _series(seed, patterns, rows_of, irregular=False, kinds=KINDS, nulls=NULLS, t0=T0):
    """one series per pattern: rows_of(pattern) rows cut by ss.mixed(pattern)"""
    rng = np.random.default_rng(seed)
    series = [ss.series_rows(rng, rows_of(p), kinds, nulls, t0=t0, irregular=irregular) for p in patterns]
    return series, [ss.mixed(p, s["times"].size) for p, s in zip(patterns, series)]


def _rows_short(p):
    return max(1100, 3 * max(p))


def _rows_long(p):
    return 2 * max(p) + 777


def _span(series):
    return int(min(s["times"][0] for s in series)), int(max(s["times"][-1] for s in series))


# ragged shards: every series is cut its own way
SHORT_PATTERNS = [[x] for x in SHORT] + [[1000, 1, 1024], [3, 1023, 33], [2, 999], [1024, 1000, 31, 32]]
# The oracle restates the reference's aggregate cursor, which keeps a record's window starts as uint16 row indices
# (engine/aggregate_cursor.go:352), so it cannot answer for segments of more than 65536 rows (DESIGN.md "Deviations").  Shards
# compared with the oracle stop at 65536 rows; longer segments are checked against the numpy model.
LONG_PATTERNS = [[x] for x in LONG if x <= 65536] + [[1000, 65536], [1, 4096, 2], [65536, 1000], [1024, 1025], [999, 8192, 3]]


@pytest.fixture(scope="module")
def short_shard():
    # no 2-row segments: their time pages are raw, which rules k_fused_cols out for the whole shard (the long shard has them)
    def rows_of(p):
        n = _rows_short(p)
        while 2 in ss.mixed(p, n):
            n += 1
        return n
    series, cuts = _series(1, [p for p in SHORT_PATTERNS if 2 not in p], rows_of)
    assert 2 not in {x for c in cuts for x in c}
    sh, sd = ss.open_shard(series, TYPES, cuts)
    yield sh, sd, series
    sh.close()


@pytest.fixture(scope="module")
def long_shard():
    series, cuts = _series(2, LONG_PATTERNS + SHORT_PATTERNS + SHORT_PATTERNS[6:13], lambda p: _rows_long(p) if max(p) > 1024 else _rows_short(p))
    sh, sd = ss.open_shard(series, TYPES, cuts)
    yield sh, sd, series
    sh.close()


# ---------------------------------------------------------------------------------------------------------------
# aggregates against the oracle
# ---------------------------------------------------------------------------------------------------------------
def _single_paths(col, const_time=True):
    if TYPES[col] == L.TYPE_FLOAT and col in (FHI, FRAW) and const_time:  # Full-header Gorilla / raw pages: the interleaved copy
        return [2, 1, 0]
    return [1, 0]


def _queries(lo, hi):
    """(interval, offset, tmin, tmax): the cadence, 7 s, 60 s, 3600 s, no interval; ranges cut inside long segments, an offset"""
    span = hi - lo
    return [(SEC, 0, lo, hi)] * (span < 20_000 * SEC) + [(7 * SEC, 0, lo, hi), (60 * SEC, 0, lo, hi), (3600 * SEC, 0, lo, hi), (0, 0, lo, hi),
            (60 * SEC, 13 * SEC, lo + span // 3 + 7, hi - span // 5), (45 * SEC, -SEC, lo + min(65536 * SEC, span // 2) - 3, hi)]


def _geometry(sh, sd, series, multi_paths, monkeypatch, tag, const_time=True):
    lo, hi = _span(series)
    n = len(series)
    for iv, off, t0, t1 in _queries(lo, hi):
        for col in (FHI, FRAW, FLO, IS8B, ICONST, BOOL, IWIDE):
            funcs = ALL6 if TYPES[col] != L.TYPE_BOOL else ["count", "min", "max", "first", "last"]
            for path in _single_paths(col, const_time):
                _agg(sh, sd, [(f, col) for f in funcs], iv, t0, t1, path, monkeypatch, f"{tag} c{col} iv={iv}", offset=off)
        for path in multi_paths if iv >= 60 * SEC or iv == 0 else [4]:  # windows below 60 s: path 4 only
            _agg(sh, sd, [("sum", FHI), ("count", FLO), ("max", IS8B), ("last", BOOL), ("first", FHI)], iv, t0, t1, path,
                 monkeypatch, f"{tag} multi iv={iv}", offset=off)
            _agg(sh, sd, [("min", ICONST), ("sum", IWIDE), ("count", FRAW)], iv, t0, t1, path, monkeypatch, f"{tag} multi ints iv={iv}", offset=off)
    iv = 60 * SEC
    for path in multi_paths + [0]:
        _agg(sh, sd, [("count", FLO), ("sum", FHI), ("max", IS8B)], iv, lo, hi, path, monkeypatch, f"{tag} where", filter=[("term", IS8B, ">", 0)])
    for path in [p for p in multi_paths if p != 5] + [0]:  # k_fused_cols takes one WHERE term at most
        _agg(sh, sd, [("sum", IS8B), ("first", FLO)], 3600 * SEC, lo, hi, path, monkeypatch, f"{tag} rpn",
             filter=[("term", FHI, "<", 100.5), ("term", BOOL, "=", 1), "or", ("term", FLO, ">=", 20.0), "and"])
    for path in _single_paths(FHI, const_time) + multi_paths[:1]:
        calls = [("sum", FHI), ("max", FHI)] if path < 4 else [("sum", FHI), ("max", IS8B), ("count", BOOL)]
        _agg(sh, sd, calls, iv, lo, hi, path, monkeypatch, f"{tag} per series", group="series")
        _agg(sh, sd, calls, 600 * SEC, lo, hi, path, monkeypatch, f"{tag} map", group="map", series_group=np.arange(n) % 3, n_groups=3)


def test_short_segments_on_every_path(short_shard, monkeypatch):
    """lengths 1 .. 1024 but 2, series cut their own way: path 5 takes the multi-column queries"""
    sh, sd, series = short_shard
    _geometry(sh, sd, series, [5, 4], monkeypatch, "short")


def test_long_segments_on_every_path(long_shard, monkeypatch):
    """lengths 2048 .. 65537 and series mixing 1000-row and 65537-row segments: path 4 takes every multi-column query"""
    sh, sd, series = long_shard
    _geometry(sh, sd, series, [4], monkeypatch, "long")


def test_irregular_times(monkeypatch):
    """Simple8b time pages rule out the interleaved copy and k_fused_cols: paths 1, 4 and 0"""
    series, cuts = _series(3, [[1, 1025], [65536], [33, 4096], [2], [1024]], lambda p: 2 * max(p) + 300, irregular=True)
    sh, sd = ss.open_shard(series, TYPES, cuts)
    lo, hi = _span(series)
    for iv in (60 * SEC, 3600 * SEC, 0):
        for col in (FHI, IS8B, BOOL):
            funcs = ALL6 if TYPES[col] != L.TYPE_BOOL else ["count", "min", "max", "first", "last"]
            for path in (1, 0):
                _agg(sh, sd, [(f, col) for f in funcs], iv, lo + 5 * SEC, hi, path, monkeypatch, f"irregular c{col} iv={iv}")
        _agg(sh, sd, [("sum", FHI), ("count", FLO), ("last", IS8B)], iv, lo, hi, 4, monkeypatch, f"irregular multi iv={iv}")
    q = AggQuery(sh, [("sum", FHI), ("count", FLO)], 60 * SEC, lo, hi, flags=L.Q_STRICT_ORDER).run()
    assert q.stats()["path"] == 4  # without OGPU_NO_COLS: the time pages alone rule path 5 out
    q.close()
    sh.close()


def test_1024_rows_take_path_5_and_1025_rows_path_4(monkeypatch):
    """the same shard with one 1025-row segment added: the longest segment decides the plan for every multi-column query"""
    patterns = [[1024], [1000, 24], [1, 1023], [1024, 1024]]
    series, cuts = _series(4, patterns, lambda p: 3072)
    for extra, path in ((None, 5), ([1025, 1], 4)):
        cc = [list(c) for c in cuts]
        if extra:
            cc[2] = extra + ss.mixed([1024], 3072 - sum(extra))
        assert max(max(c) for c in cc) == (1025 if extra else 1024)
        sh, sd = ss.open_shard(series, TYPES, cc)
        lo, hi = _span(series)
        for iv in (60 * SEC, 7 * SEC, 0):
            _agg(sh, sd, [("sum", FHI), ("count", FLO), ("max", IS8B), ("first", BOOL)], iv, lo, hi, path, monkeypatch,
                 f"1024/1025 iv={iv}")
            _agg(sh, sd, [("count", FHI), ("sum", IS8B)], iv, lo + 100 * SEC, hi, path, monkeypatch, f"1024/1025 where iv={iv}",
                 filter=[("term", FRAW, "<", 1.0)])
        sh.close()


def test_chunk_plans_cut_between_series_of_different_lengths(long_shard, monkeypatch):
    """OGPU_CHUNK_SERIES=32: chunks of 32 series on a ragged shard whose series hold 1 .. 65537-row segments"""
    sh, sd, series = long_shard
    lo, hi = _span(series)
    monkeypatch.setenv("OGPU_CHUNK_SERIES", "32")
    assert len(series) > 32
    for path in (2, 1, 0):
        _agg(sh, sd, [("sum", FHI), ("count", FHI), ("min", FHI)], 60 * SEC, lo, hi, path, monkeypatch, "chunks")
        _agg(sh, sd, [("last", FHI)], 3600 * SEC, lo, hi, path, monkeypatch, "chunks per series", group="series")
    _agg(sh, sd, [("sum", IS8B), ("max", FLO), ("count", BOOL)], 60 * SEC, lo, hi, 4, monkeypatch, "chunks multi")
    _agg(sh, sd, [("sum", FHI), ("count", IS8B)], 600 * SEC, lo, hi, 4, monkeypatch, "chunks map", group="map",
         series_group=np.arange(len(series)) % 5, n_groups=5)


# ---------------------------------------------------------------------------------------------------------------
# k_fused_il: the folded path on regular shards of long segments, lane drift, the window cap, eligibility caps
# ---------------------------------------------------------------------------------------------------------------
def _regular(seed, n_series, lengths, kind, t0=T0):
    rng = np.random.default_rng(seed)
    series = [ss.series_rows(rng, sum(lengths), [kind], t0=t0) for _ in range(n_series)]
    return ss.open_shard(series, [L.TYPE_FLOAT], [list(lengths)] * n_series) + (series,)


@pytest.mark.parametrize("length", [33, 1001, 1025, 4096, 65535])
def test_folded_path_on_regular_shards(length, monkeypatch):
    """every series cut the same way: paths 3 and 2 on Gorilla and raw pages"""
    for kind in ("f_hi", "f_raw"):
        sh, sd, series = _regular(length, 34, [length] * 3, kind)
        lo, hi = _span(series)
        for iv, t0, t1 in ((60 * SEC, lo, hi), (7 * SEC, lo + length * SEC + 3, hi - 1), (3600 * SEC, lo, hi), (0, lo, hi)):
            for calls in ([(f, 0) for f in ALL6], [("sum", 0), ("count", 0)], [("max", 0)], [("first", 0), ("last", 0)]):
                for path in (3, 2):
                    st = _agg(sh, sd, calls, iv, t0, t1, path, monkeypatch, f"regular {length} {kind} {calls} iv={iv}")
                    assert st["general_segments"] == 0 and st["il_state"] == 1
        sh.close()


def _drift_shard(n_series, kind, seed):
    """One series is a single 65535-row segment; the others one 3-row or 1000-row segment over the same time range (const-delta
    pages of different cadences), so the shard is regular and aligned and k_fused_il folds it: the long lane shares its lane
    group with 1000-row lanes that finish long before it.  The 3-row segments step by more than 2^40 ns, which the copy does not
    take: they are left to the general kernel."""
    span = 65534 * 999 * 1_000_000  # divisible by 65534, 999 and 2
    rng = np.random.default_rng(seed)
    series, lens = [], []
    for s in range(n_series):
        n = 65535 if s == n_series // 2 else (3 if s % 2 else 1000)
        t = T0 + np.arange(n, dtype=np.int64) * (span // (n - 1))
        rows = ss.series_rows(rng, n, [kind])
        rows["times"] = t
        series.append(rows); lens.append([n])
    return ss.open_shard(series, [L.TYPE_FLOAT], lens) + (series,)


@pytest.mark.parametrize("n_series", [40, 32])
@pytest.mark.parametrize("kind", ["f_raw", "f_lo"])
def test_drift_of_one_long_lane_among_short_lanes(n_series, kind, monkeypatch):
    """one 65535-row lane among 1000-row lanes in a lane group (f_raw: packed lanes, f_lo: Gorilla lanes)"""
    sh, sd, series = _drift_shard(n_series, kind, 7)
    lo, hi = _span(series)
    for iv in (60 * SEC, 3600 * SEC, 0):
        for calls in ([(f, 0) for f in ALL6], [("sum", 0), ("count", 0), ("max", 0)], [("first", 0), ("last", 0)]):
            for path in (3, 2):
                st = _agg(sh, sd, calls, iv, lo, hi, path, monkeypatch, f"drift {kind} {calls} iv={iv}")
                n_il = n_series - n_series // 2  # the 1000-row lanes and the long one; 3-row segments go to the general kernel
                assert st["general_segments"] == n_series // 2
                if kind == "f_raw":
                    assert st["il_packed_segments"] == n_il
                else:
                    assert st["il_packed_segments"] < n_il
    _agg(sh, sd, [("min", 0), ("last", 0)], 60 * SEC, lo, hi, 2, monkeypatch, "drift per series", group="series")
    sh.close()


def test_window_cap_of_the_folding_warp(monkeypatch):
    """A segment folded in the warp spans at most OG_IL_WCAP = 24 windows.  1440 rows at 1 s from a window boundary span 24
    windows of 60 s: no per-series cells.  1441 and 4096 rows span more: per-series cells.  All equal the oracle."""
    t0 = T0 + (60 * SEC - T0 % (60 * SEC))  # a 60 s window boundary
    for length, spill in ((1440, 0), (1441, 1), (4096, 1), (65536, 1)):
        sh, sd, series = _regular(length, 40, [length, length], "f_hi", t0=t0)
        lo, hi = _span(series)
        for calls in ([("sum", 0), ("count", 0)], [(f, 0) for f in ALL6]):
            st = _agg(sh, sd, calls, 60 * SEC, lo, hi, 3, monkeypatch, f"wcap {length} {calls}")
            assert st["per_series_cells_used"] == spill, (length, st["per_series_cells_used"])
        sh.close()


def _pool_used():
    from test_gpu_device_memory import _pool_used as used
    return used()


def test_eligibility_caps_of_the_interleaved_copy(monkeypatch, capsys):
    """rows in [2, 2^22) go into the copy: a 2^22 - 1-row segment does, a 2^22-row one and one-row segments are left to the
    general kernel.  Checked against the numpy model.  Path 0 sizes its tile as 32 segments of the longest segment: the device
    memory its first run takes is recorded here at 2^22 rows."""
    rng = np.random.default_rng(22)
    big = 1 << 22
    series = [ss.series_rows(rng, big - 1, ["f_hi"]), ss.series_rows(rng, big, ["f_hi"]), ss.series_rows(rng, 3, ["f_hi"])]
    cuts = [[big - 1], [big], [1, 1, 1]]
    sh, sd = ss.open_shard(series, [L.TYPE_FLOAT], cuts)
    lo, hi = _span(series)
    models = {iv: ss.window_model(series, 0, L.TYPE_FLOAT, iv, 0, lo, hi, [0, 0, 0]) for iv in (3600 * SEC, 0)}
    for calls, iv in (([("sum", 0), ("count", 0), ("max", 0)], 3600 * SEC), ([("first", 0), ("last", 0), ("min", 0)], 0)):
        for path in (2, 1, 0):
            q = AggQuery(sh, calls, iv, lo, hi, flags=FLAGS[path])
            before = _pool_used()
            q.run()
            grown = _pool_used() - before
            st = q.stats()
            assert st["path"] == path
            if path == 2:
                assert st["general_segments"] == 4, st["general_segments"]  # the 2^22-row segment and three one-row segments
            ss.check_against_model(q.dense_host(), calls, models[iv], L.TYPE_FLOAT, f"caps {calls} path {path}")
            q.close()
    tile = 32 * big * (9 + 8 + 1)  # values + validity of one column, times, keep flags
    with capsys.disabled():
        print(f"\npath 0 at {big} rows per segment: {grown / 2**30:.2f} GiB of device memory for the query (tile {tile / 2**30:.2f} GiB)")
    assert grown >= tile
    sh.close()


# ---------------------------------------------------------------------------------------------------------------
# invariance under re-cutting: the same rows, any cut, the same answers (numpy model, no oracle)
# ---------------------------------------------------------------------------------------------------------------
RECUT = {"1000": [1000], "1024": [1024], "4096": [4096], "65535": [65535], "mixed": [1000, 65537, 3, 4096, 1]}
RECUT_KINDS = ["f_hi", "f_raw", "i_s8b", "bool", "i_const"]


def test_answers_do_not_depend_on_the_cut(monkeypatch):
    rng = np.random.default_rng(99)
    n, n_series = 100_003, 12
    series = [ss.series_rows(rng, n, RECUT_KINDS, [0, 0, 0.1, 0.2, 0]) for _ in range(n_series)]
    types = ss.types_of(RECUT_KINDS)
    lo, hi = _span(series)
    queries = [(60 * SEC, 0, lo, hi, "all"), (3600 * SEC, 0, lo, hi, "series"), (7 * SEC, 2 * SEC, lo + 70_000 * SEC + 1, hi - 3 * SEC, "all"),
               (0, 0, lo + 999 * SEC, hi, "all"), (600 * SEC, 0, lo, lo + 65537 * SEC, "series")]
    models, first = {}, {}
    for cut, pattern in RECUT.items():
        sh, _sd = ss.open_shard(series, types, [ss.mixed(pattern, n)] * n_series)
        for qi, (iv, off, t0, t1, group) in enumerate(queries):
            groups = [0] * n_series if group == "all" else list(range(n_series))
            for col, typ in enumerate(types):
                key = (qi, col)
                if key not in models:
                    models[key] = ss.window_model(series, col, typ, iv, off, t0, t1, groups)
                funcs = ["count", "min", "max", "first", "last"] + ([] if typ == L.TYPE_BOOL else ["sum"])
                paths = [1, 0] + ([2] + ([3] if group == "all" else []) if typ == L.TYPE_FLOAT else [])
                for path in paths:
                    q = AggQuery(sh, [(f, col) for f in funcs], iv, t0, t1, offset=off, group=group, flags=FLAGS[path]).run()
                    assert q.stats()["path"] == path, (cut, path)
                    d = q.dense_host()
                    q.close()
                    label = f"cut {cut} q{qi} c{col} path {path}"
                    ss.check_against_model(d, [(f, col) for f in funcs], models[key], typ, label)
                    bits = [np.asarray(c["values"]).view(np.uint64) if f != "sum" or typ != L.TYPE_FLOAT else None for f, c in zip(funcs, d["cols"])]
                    times = [None if c["times"] is None else np.asarray(c["times"]) for c in d["cols"]]
                    if (qi, col) in first:
                        b0, t0_ = first[(qi, col)]
                        for k in range(len(funcs)):
                            if bits[k] is not None:
                                assert np.array_equal(bits[k], b0[k]), f"{label} {funcs[k]} differs from the first cut"
                            if times[k] is not None:
                                assert np.array_equal(times[k][models[key]["valid"]], t0_[k][models[key]["valid"]]), label
                    else:
                        first[(qi, col)] = (bits, times)
            multi = [("sum", 2), ("count", 3), ("max", 0), ("first", 1)]
            for path in ([5] if cut in ("1000", "1024") else []) + [4]:
                with monkeypatch.context() as m:
                    if path == 4:
                        m.setenv("OGPU_NO_COLS", "1")
                    q = AggQuery(sh, multi, iv, t0, t1, offset=off, group=group, flags=L.Q_STRICT_ORDER).run()
                    assert q.stats()["path"] == path
                    d = q.dense_host()
                    q.close()
                for k, (f, col) in enumerate(multi):
                    one = dict(n_buckets=d["n_buckets"], start=d["start"], cols=[d["cols"][k]])
                    ss.check_against_model(one, [(f, col)], models[(qi, col)], types[col], f"cut {cut} q{qi} multi {f} path {path}", multi=True)
        sh.close()


# ---------------------------------------------------------------------------------------------------------------
# materialisation
# ---------------------------------------------------------------------------------------------------------------
DECODE_LENGTHS = SHORT + LONG[:-1]  # up to 65536 rows: descending materialisation takes them all


@pytest.fixture(scope="module")
def decode_shard():
    rng = np.random.default_rng(5)
    series = [ss.series_rows(rng, n, KINDS, NULLS, irregular=bool(i % 2)) for i, n in enumerate(DECODE_LENGTHS)]
    sh, sd = ss.open_shard(series, TYPES, [[n] for n in DECODE_LENGTHS])
    yield sh, sd
    sh.close()


def _pages(sh):
    ex = sh.export()
    return ex, [[ex["data"][int(o):int(o) + int(z)] for o, z in zip(ex["page_off"][c], ex["page_len"][c])] for c in range(ex["page_off"].shape[0])]


def test_decode_segment_ascending_and_descending(decode_shard):
    sh, _sd = decode_shard
    _ex, pages = _pages(sh)
    for g, n in enumerate(DECODE_LENGTHS):
        want_t = oracle.time_page_decode(pages[-1][g], cap=n + 8)
        for desc in (False, True):
            r = (lambda a: np.ascontiguousarray(a[::-1])) if desc else (lambda a: a)
            rec = sh.decode_segment(g, descending=desc)
            assert rec["rows"] == n and np.array_equal(rec["times"], r(want_t)), (n, desc)
            for c, ty in enumerate(TYPES):
                v, ok = oracle.field_page_decode(ty, pages[c][g], cap=n + 8)
                col = rec["cols"][c]
                assert np.array_equal(col["valid"], r(ok)), (n, c, desc)
                assert col["nil_count"] == int((~ok).sum()) and col["len"] == n
                assert np.ascontiguousarray(col["values"]).tobytes() == np.ascontiguousarray(r(v)).tobytes(), (n, c, desc)


def test_descending_materialisation_refuses_segments_above_65536_rows():
    """one 65537-row segment in the shard: every segment is refused descending (the reversal's bitmap holds 65536 rows), ascending
    still decodes, and ScanCursor does the same"""
    rng = np.random.default_rng(6)
    series = [ss.series_rows(rng, 1000, KINDS, NULLS), ss.series_rows(rng, 65537, KINDS, NULLS), ss.series_rows(rng, 33, KINDS, NULLS)]
    sh, _sd = ss.open_shard(series, TYPES, [[1000], [65537], [33]])
    _ex, pages = _pages(sh)
    for g, rows in enumerate(series):
        with pytest.raises(L.OgpuError) as ei:
            sh.decode_segment(g, descending=True)
        assert ei.value.status == L.OG_E_UNSUPPORTED and "65536" in str(ei.value)
        rec = sh.decode_segment(g)
        assert np.array_equal(rec["times"], rows["times"])
        for c, ty in enumerate(TYPES):
            v, ok = oracle.field_page_decode(ty, pages[c][g], cap=rows["times"].size + 8)
            assert np.array_equal(rec["cols"][c]["valid"], ok)
            assert np.ascontiguousarray(rec["cols"][c]["values"]).tobytes() == np.ascontiguousarray(v).tobytes()
    lo, hi = _span(series)
    with pytest.raises(L.OgpuError) as ei:
        list(ScanCursor(sh, lo, hi, ascending=False))
    assert ei.value.status == L.OG_E_UNSUPPORTED
    got = list(ScanCursor(sh, lo + 10 * SEC, hi))
    assert [r["rows"] for r in got] == [990, 65527, 23]
    assert np.array_equal(got[1]["times"], series[1]["times"][10:])
    sh.close()


def test_decode_column_device_over_mixed_lengths(decode_shard):
    sh, _sd = decode_shard
    ex, pages = _pages(sh)
    nc, nseg = len(TYPES), len(DECODE_LENGTHS)
    for a, b in ((0, nseg), (5, 13), (14, 17), (nseg - 1, nseg)):
        stride = 8 * max(DECODE_LENGTHS[a:b]) + 24  # the caller's stride, wider than any segment
        for c in range(nc + 1):
            vals = torch.full(((b - a) * stride,), 0xA5, dtype=torch.uint8, device="cuda")
            rows = torch.full((b - a,), -1, dtype=torch.int32, device="cuda")
            L.check(L.lib().og_decode_column_device(sh.h, c, a, b, vals.data_ptr(), stride, rows.data_ptr()), "og_decode_column_device")
            hv, hr = vals.cpu().numpy(), rows.cpu().numpy()
            for k, g in enumerate(range(a, b)):
                n = DECODE_LENGTHS[g]
                if c == nc:
                    want = oracle.time_page_decode(pages[c][g], cap=n + 8).view(np.uint8)
                    assert hr[k] == n, (c, g)
                else:
                    v, ok = oracle.field_page_decode(TYPES[c], pages[c][g], cap=n + 8)
                    want = np.ascontiguousarray(v).view(np.uint8)
                    assert hr[k] == int(ok.sum()), (c, g, hr[k], int(ok.sum()))
                got = hv[k * stride:(k + 1) * stride]
                assert np.array_equal(got[:want.size], want), (c, g)
                assert (got[want.size:] == 0xA5).all(), (c, g)  # nothing written past the segment's values
    vals = torch.full((64,), 7, dtype=torch.uint8, device="cuda")
    rows = torch.full((4,), -1, dtype=torch.int32, device="cuda")
    L.check(L.lib().og_decode_column_device(sh.h, 0, 3, 3, vals.data_ptr(), 8, rows.data_ptr()), "empty range")
    assert (vals.cpu().numpy() == 7).all() and (rows.cpu().numpy() == -1).all()
    for col, s0, s1 in ((nc + 1, 0, 1), (0, 2, 1), (0, 0, nseg + 1), (0, nseg + 1, nseg + 1)):
        assert L.lib().og_decode_column_device(sh.h, col, s0, s1, vals.data_ptr(), 8, rows.data_ptr()) == L.OG_E_INVAL, (col, s0, s1)


# ---------------------------------------------------------------------------------------------------------------
# write, merge, downsample
# ---------------------------------------------------------------------------------------------------------------
def test_tssp_write_of_long_segments():
    import tssp_write_model as M
    from test_gpu_tssp_write import _check_crcs, _same_answers, make_chunks, shard_desc
    cols = [("a_fhi", "f_hi", 0.05), ("b_fraw", "f_raw", 0), ("c_is8b", "i_s8b", 0.3), ("d_bool", "bool", 0.5), ("e_iconst", "i_const", 0)]
    chunks = make_chunks(31, 4, cols, lambda rng, s: [[4096, 65535], [65535], [3, 4096, 1, 4096], [65536, 2]][s], ("const", "s8b"))
    sh = Shard.open_desc(shard_desc(chunks, seed=4))
    try:
        got = write_tssp(sh, "long")
        assert got == M.build(chunks, b"long")
        _check_crcs(got)
        back = Shard.open_tssp(got)
        try:
            assert _same_answers(sh, back, [ty for _n, ty, _p, _r in chunks[0]["columns"]], filter_col=2) >= 10
        finally:
            back.close()
    finally:
        sh.close()


def _compare_files(sh, files, calls, iv, tmin, tmax, seg_rows, where=None, **kw):
    """the merged shard against oracle_files.scan_aggregate_files, whose ordered records are the file's seg_rows-row segments"""
    import oracle_files
    names = sorted({n for f, _ in files for s_ in f.values() for n in s_["cols"]})
    flt = [("term", it[0], it[1], it[2]) for it in where] if where else None
    q = AggQuery(sh, calls, iv, tmin, tmax, filter=flt, **kw).run()
    got = q.dense_host()
    ref, _sids = oracle_files.scan_aggregate_files(files, q, [(names[it[0]], it[1], it[2]) for it in where] if where else None,
                                                   seg_rows=seg_rows)
    q.close()
    for k, (f, c) in enumerate(calls):
        rv = ref["cols"][k]["valid"].astype(bool)
        assert np.array_equal(got["cols"][k]["valid"].astype(bool), rv), (f, c, iv, kw)
        g, r = got["cols"][k]["values"].view(np.uint64)[rv], ref["cols"][k]["values"][rv]
        if f == "sum" and got["cols"][k]["type"] == L.TYPE_FLOAT:  # merged series: float sums within 1e-12 (DESIGN.md "Deviations")
            gf, rf = g.view(np.float64), r.view(np.float64)
            assert np.all(np.abs(gf - rf) <= 1e-12 * np.maximum(1.0, np.abs(rf))), (f, c, iv, kw)
        else:
            assert np.array_equal(g, r), (f, c, iv, kw)
        if got["cols"][k]["times"] is not None and f in ("min", "max", "first", "last"):
            assert np.array_equal(got["cols"][k]["times"][rv], ref["cols"][k]["times"][rv]), (f, c, iv, kw)


@pytest.mark.parametrize("batch", [None, "1500"])
def test_merge_of_an_ordered_file_of_4096_row_segments(batch, monkeypatch):
    """the merge rewrites overlapped spans into 1000-row segments and keeps the other 4096-row segments: series of mixed lengths"""
    from test_gpu_out_of_order import _check_rows, _file_desc, _model, _random_files
    files = _random_files(41, n_series=9, rows=13000)
    if batch:
        monkeypatch.setenv("OGPU_MERGE_BATCH_ROWS", batch)
    sh = Shard.open_files([(_file_desc(f, seg_rows=4096 if not ooo else 1000), ooo) for f, ooo in files])
    monkeypatch.delenv("OGPU_MERGE_BATCH_ROWS", raising=False)
    _check_rows(sh, _model(files))
    ex = sh.export()
    lens = {int(oracle.time_page_decode(ex["data"][int(o):int(o) + int(z)], cap=5000).size) for o, z in zip(ex["page_off"][-1], ex["page_len"][-1])}
    assert 4096 in lens and 1000 in lens, sorted(lens)
    tmin = min(int(s["times"][0]) for f, _ in files for s in f.values())
    tmax = max(int(s["times"][-1]) for f, _ in files for s in f.values())
    names = sorted({n for f, _ in files for s in f.values() for n in s["cols"]})
    fv, iv_, bv = names.index("fv"), names.index("iv"), names.index("bv")
    for iv in (60 * SEC, 3600 * SEC, 0):
        _compare_files(sh, files, [(f, fv) for f in ALL6], iv, tmin, tmax, 4096, flags=L.Q_STRICT_ORDER)
        _compare_files(sh, files, [("sum", iv_), ("count", bv), ("max", fv)], iv, tmin + 4000 * SEC + 3, tmax, 4096, flags=L.Q_STRICT_ORDER)
        _compare_files(sh, files, [("last", iv_)], iv, tmin, tmax, 4096, group="series", flags=L.Q_STRICT_ORDER)
    sh.close()


def test_downsample_of_long_segments():
    from test_gpu_downsample_shard import _check, _model
    kinds = ["f_hi", "f_lo", "i_s8b", "bool"]
    rng = np.random.default_rng(12)
    series = [ss.series_rows(rng, n, kinds, [0, 0.2, 0.1, 0.3]) for n in (70_000, 65_537, 9_000)]
    types = ss.types_of(kinds)
    d = ss.shard_desc(series, types, [ss.mixed([4096], 70_000), [65537], [1000, 8000]])
    sh = Shard.open_desc(d)
    fields = [(f"c{c}", t) for c, t in enumerate(types)]
    ops = {L.TYPE_FLOAT: ALL6, L.TYPE_INT: ["sum", "count", "min", "last"], L.TYPE_BOOL: ["count", "first", "max"]}
    lo, hi = _span(series)
    for interval, tmin, tmax in ((60 * SEC, lo, hi), (7 * SEC, lo + 3 * SEC, lo + 66_000 * SEC)):
        want_cols, model = _model(d, fields, ops, interval, tmin, tmax)
        ds = sh.downsample_shard(interval, tmin, tmax, ops)
        _check(ds, want_cols, model)
        ds.close()
    sh.close()
