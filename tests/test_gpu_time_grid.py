"""Window arithmetic on every aggregate path, away from the one-second grid.

Which rows fall in the query range and which window each row belongs to is computed five separate ways: on the host
(og_query_create), by k_fused_il (udiv_est estimates, a Bresenham step of the next window's first row, row countdowns, the
window-skip loop, the fold limit of OG_IL_WCAP windows per segment), by k_fused_cols (the same closed forms, written out
again), by the row-time compares of the general, multi-column and tile kernels, and by the edge stitch.  Each case below
names the arithmetic it aims at and runs on every path that can serve it, asserting og_stats.path:

    3  k_fused_il, folded             default
    2  k_fused_il, per-series cells   OG_Q_STRICT_ORDER, group="series", group="map", or lanes on different grids
    1  general fused kernel           OG_Q_NO_FAST, int and bool columns, or no segment k_fused_il takes
    0  materialisation tile           OG_Q_NO_FUSED
    5  k_fused_cols                   one WHERE term
    4  k_fused_multi                  two WHERE terms, or one under OGPU_NO_COLS

Every answer is compared with the CPU oracle (run_both's rules: bitwise under the strict order, float sums within
SUM_RTOL otherwise) and with the time-geometry model of time_grid.py: counts exactly, min/max/first/last and their times
bitwise, float sums against math.fsum within SUM_RTOL.  The WHERE terms keep every row, so the model's row sets hold
on paths 4 and 5 too."""
from collections import Counter
from dataclasses import dataclass, field

import numpy as np
import pytest

import oracle
import time_grid as tg
from opengemini_b200 import AggQuery, Shard
from opengemini_b200 import _lib as L
from test_gpu_parity import SUM_RTOL, _bits, compare_dense

pytestmark = pytest.mark.gpu

T0 = 1_700_000_000_000_000_000
SEC = 1_000_000_000
DAY = 86_400 * SEC
OPEN = (tg.MIN_TIME, tg.MAX_TIME)
ALL6 = ["count", "sum", "min", "max", "first", "last"]
PRIME = 999_999_937

# columns of every shard: 0 G-hi floats and 1 G-lo floats, both without nulls and with values distinct across the shard (the
# model's selectors then have one answer), 2 G-lo floats with nulls, 3/4 ints without/with nulls, 5/6 bools without/with nulls
COLS = [("ghi", L.TYPE_FLOAT), ("glo", L.TYPE_FLOAT), ("glo_nulls", L.TYPE_FLOAT), ("int", L.TYPE_INT),
        ("int_nulls", L.TYPE_INT), ("bool", L.TYPE_BOOL), ("bool_nulls", L.TYPE_BOOL)]
DISTINCT = (0, 1)
KEEP = ("term", 0, ">", 0.0)       # every value is >= 100: the WHERE keeps every row
KEEP2 = ("term", 0, "<", 1000.0)
OG_COLS_MAXMINE = 4


@pytest.fixture(scope="module", autouse=True)
def _device():
    Shard.init(0)


@dataclass
class Case:
    target: str                      # the arithmetic the case aims at
    series: list                     # [(t0, dt, rows)]
    interval: int
    offset: int = 0
    tmin: int = OPEN[0]
    tmax: int = OPEN[1]
    rows_per_seg: int = 1000
    default_path: int = 3            # path of the default query: 2 when lanes do not share a grid, 1 when k_fused_il takes nothing
    stats: dict = field(default_factory=dict)  # og_stats of the default sum/count/max query


def _n(t0, dt, rows, n=40):
    return [(t0, dt, rows)] * n


Y365 = 365 * DAY
T_Y = T0 - T0 % Y365 + Y365 - 1500   # 1500 ns before a 365-day boundary
T_Y62 = (1 << 62) - (1 << 62) % Y365 - 1500
W10 = 10 * SEC

CASES = {
    # ---- cadences ----
    "cadence_1ns": Case("1 ns rows, 10 ns windows: udiv_est on tiny divisors, whole windows of ten rows", _n(T0, 1, 1500), 10),
    "cadence_7ns": Case("7 ns rows, 10 ns windows offset by 1 ns: the Bresenham carry adds a row to some windows", _n(T0 + 3, 7, 1500), 10, 1),
    "cadence_prime": Case("999 999 937 ns rows, 60 s windows: boundaries fall between rows at a drifting phase", _n(T0, PRIME, 1500), 60 * SEC),
    "cadence_3s": Case("3 s rows, 10 s windows offset by -1 ns", _n(T0, 3 * SEC, 1500), W10, -1),
    "cadence_90s_windows_60s": Case("cadence longer than the interval: the window-skip loop runs and every third window is empty",
                                    _n(T0, 90 * SEC, 1500), 60 * SEC),
    "cadence_2^40_edge": Case("dt = 2^40 - 1 (k_fused_il) next to dt = 2^40 (general kernel) in one shard, 3*2^40+5 ns windows",
                              [(T0, (1 << 40) - 1 + (s % 2), 100) for s in range(40)], 3 * (1 << 40) + 5, default_path=2),
    # ---- intervals ----
    "interval_1ns": Case("1 ns windows over 1 ns rows: one row per window, 1500 buckets", _n(T0, 1, 1500), 1),
    "interval_eq_dt": Case("interval == dt: one row per window, boundaries on rows", _n(T0, PRIME, 1500), PRIME),
    "interval_dt_minus_1": Case("interval == dt - 1: the boundary moves 1 ns closer to the next row every window",
                                _n(T0, PRIME, 1500), PRIME - 1),
    "interval_dt_plus_1": Case("interval == dt + 1: step_r = 1, the carry fires once the drift adds up", _n(T0, PRIME, 1500), PRIME + 1),
    "interval_10ns_cadence_3ns": Case("10 ns windows over 3 ns rows: 3 or 4 rows a window", _n(T0, 3, 1500), 10),
    "interval_365d_cadence_1ns": Case("365-day windows over 1 ns rows across a boundary: quotients >= 2^50 take the exact "
                                      "division, step_q clamps at 2^32-1", _n(T_Y, 1, 3000), Y365),
    "interval_wider_than_shard": Case("1 ms windows over 10.5 us of data: one bucket", _n(T0, 7, 1500), 1_000_000),
    "interval_0": Case("no interval, open range: one bucket spanning the shard", _n(T0, 7, 1500), 0),
    # ---- offsets ----
    "offset_1ns": Case("offset 1 ns", _n(T0, SEC, 1500), 60 * SEC, 1),
    "offset_interval_minus_1": Case("offset interval - 1", _n(T0, SEC, 1500), 60 * SEC, 60 * SEC - 1),
    "offset_minus_1": Case("offset -1 ns", _n(T0, 7, 1500), 60, -1),
    "offset_interval_plus_3": Case("offset interval + 3: more than one interval", _n(T0, 7, 1500), 60, 63),
    "offset_minus_2_intervals_minus_5": Case("offset -2 * interval - 5", _n(T0, 7, 1500), 60, -125),
    # ---- range ends ----
    "range_rows_outside": Case("tmin a row - 1 ns, tmax a row + 1 ns", _n(T0, 7, 1500), 60, 0, T0 + 7 * 100 - 1, T0 + 7 * 1400 + 1),
    "range_rows_inside": Case("tmin a row + 1 ns, tmax a row - 1 ns", _n(T0, 7, 1500), 60, 0, T0 + 7 * 100 + 1, T0 + 7 * 1400 - 1),
    "range_on_rows": Case("tmin and tmax on rows", _n(T0, 7, 1500), 60, 0, T0 + 7 * 100, T0 + 7 * 1400),
    "range_boundaries_minus_1": Case("tmin and tmax a window boundary - 1 ns", _n(T0, 7, 1500), 60, 0, T0 + 600 - 1, T0 + 9000 - 1),
    "range_boundaries_plus_1": Case("tmin and tmax a window boundary + 1 ns", _n(T0, 7, 1500), 60, 0, T0 + 600 + 1, T0 + 9000 + 1),
    "range_between_two_rows": Case("a range that holds no row", _n(T0, 7, 1500), 60, 0, T0 + 7 * 100 + 1, T0 + 7 * 101 - 1),
    "range_one_row": Case("tmin == tmax on a row", _n(T0, 7, 1500), 60, 0, T0 + 7 * 555, T0 + 7 * 555),
    # ---- fold limit: one segment per series, aligned 10 s windows ----
    "fold_24_windows": Case("segments of 240 rows at 1 s touch exactly OG_IL_WCAP = 24 windows: folded in the warp",
                            _n(T0, SEC, 240, 64), W10, stats=dict(per_series_cells_used=0)),
    "fold_25_windows": Case("segments of 250 rows touch 25 windows: one past the fold limit, per-series cells",
                            _n(T0, SEC, 250, 64), W10, stats=dict(per_series_cells_used=1)),
    # ---- shifted grids ----
    "shifted_grids": Case("series whose t0 differ by 13 ns steps over a 1 000 003 ns cadence: lanes share groups, not grids",
                          [(T0 + 13 * s, 1_000_003, 1500) for s in range(40)], 7 * SEC // 100, default_path=2),
    # ---- times far from the epoch ----
    "near_2^62_1ns": Case("1 ns rows just below 2^62, 7 ns windows", _n((1 << 62) - 700, 1, 1500), 7),
    "near_minus_2^62_7ns": Case("7 ns rows across -2^62, 60 ns windows offset by 3", _n(-(1 << 62) - 7 * 700, 7, 1500), 60, 3),
    "near_2^62_365d": Case("1 ns rows across the last 365-day boundary below 2^62", _n(T_Y62, 1, 3000), Y365),
    # ---- the int64 limits (the CPU model shows these grids unclamped) ----
    "max_time_bounded": Case("rows up to MAX_TIME, tmax keeps the last window unclamped", _n(tg.MAX_TIME - 7 * 1499, 7, 1500), 100,
                             0, OPEN[0], tg.MAX_TIME - 200),
    "max_time_last_whole_window": Case("the last row ends the last whole window below MAX_TIME: only the empty window after it "
                                       "is clamped", _n(tg.MAX_TIME - tg.MAX_TIME % 100 - 1 - 7 * 1499, 7, 1500), 100),
    "min_time_first_boundary": Case("the first row on the first window boundary above MIN_TIME",
                                    _n(tg.MIN_TIME + (-tg.MIN_TIME) % 100, 7, 1500), 100),
}

_SHARDS = {}


class GShard:
    def __init__(self, case, seed=0):
        rng = np.random.default_rng(seed)
        total = sum(n for _, _, n in case.series)
        glo_pool = 100.0 + rng.permutation(total).astype(np.float64) / 1024.0
        self.times, self.values = [], {c: [] for c in range(len(COLS))}
        pages = {c: [] for c in range(len(COLS))}
        tpages, tmins, tmaxs, ssb, k = [], [], [], [0], 0
        for t0, dt, n in case.series:
            t = np.array([t0 + i * dt for i in range(n)], np.int64)
            i = np.arange(n)
            cols = [100.0 + rng.random(n), glo_pool[k:k + n], 100.0 + (i % 16) * 0.25,
                    np.cumsum(rng.integers(-50, 51, n)).astype(np.int64), np.cumsum(rng.integers(-50, 51, n)).astype(np.int64),
                    rng.integers(0, 2, n).astype(np.uint8), rng.integers(0, 2, n).astype(np.uint8)]
            k += n
            self.times.append([int(x) for x in t])
            for c, v in enumerate(cols):
                self.values[c].append(v.tolist())
            for a in range(0, n, case.rows_per_seg):
                sl = slice(a, a + case.rows_per_seg)
                for c, (_name, typ) in enumerate(COLS):
                    valid = (i[sl] % NULL_EVERY[c][0] != NULL_EVERY[c][1]).astype(np.uint8) if c in NULL_EVERY else None
                    pages[c].append(oracle.field_page_encode(typ, cols[c][sl], valid))
                tpages.append(oracle.time_page_encode(t[sl])); tmins.append(int(t[sl][0])); tmaxs.append(int(t[sl][-1]))
            ssb.append(len(tpages))
        blob, pos, cols_desc = [], 0, []
        for c, (name, typ) in enumerate(COLS):
            offs, lens = [], []
            for p in pages[c]:
                offs.append(pos); lens.append(p.size); blob.append(p); pos += p.size
            cols_desc.append((name, typ, offs, lens))
        toffs, tlens = [], []
        for p in tpages:
            toffs.append(pos); tlens.append(p.size); blob.append(p); pos += p.size
        self.n_series = len(case.series)
        self.sh = Shard.open(np.concatenate(blob), np.arange(1, self.n_series + 1), ssb, tmins, tmaxs, cols_desc, toffs, tlens)
        self.sd = oracle.shard_desc_from_export(self.sh.export())
        self.tmin, self.tmax = min(tmins), max(tmaxs)


@pytest.fixture(scope="module")
def shards():
    yield _SHARDS
    for g in _SHARDS.values():
        g.sh.close()
    _SHARDS.clear()


def _shard(shards, name):
    if name not in shards:
        shards[name] = GShard(CASES[name])
    return shards[name]


def _model(g, case, query_grid=False, tmin=None, tmax=None):
    tmin = case.tmin if tmin is None else tmin
    tmax = case.tmax if tmax is None else tmax
    grid = tg.grid(case.interval, case.offset, tmin, tmax, g.tmin, g.tmax, query_grid)
    assert not grid.clamped
    return grid, tg.bucket_rows(g.times, grid, case.interval, case.offset)


_EXPECTED = {}
NULL_EVERY = {2: (7, 3), 4: (5, 1), 6: (6, 2)}  # column: (m, k), row j of a series is null when j % m == k


def _expected(rows, g, col):
    key = (id(rows), col)
    if key not in _EXPECTED:
        valid = None
        if col in NULL_EVERY:
            m, k = NULL_EVERY[col]
            valid = [[j % m != k for j in range(len(ts))] for ts in g.times]
        _EXPECTED[key] = (rows, tg.expected(rows, g.times, g.values[col], valid))
    return _EXPECTED[key][1]


def check_model(gpu, grid, rows, g, calls, label):
    """gpu: one-group dense record.  Calls on a DISTINCT column are checked in full, counts and sums on any column."""
    assert gpu["n_buckets"] == grid.n_buckets and gpu["start"] == grid.start, f"{label}: grid {gpu['start']}+{gpu['interval']}x{gpu['n_buckets']}"
    multi = len(calls) > 1
    for k, (func, col) in enumerate(calls):
        if func not in ("count", "sum") and col not in DISTINCT:
            continue
        typ = COLS[col][1]
        want = _expected(rows, g, col)
        c = gpu["cols"][k]
        valid = np.asarray(c["valid"]).astype(bool)
        assert sorted(np.flatnonzero(valid).tolist()) == sorted(want), f"{label} call {k} ({func}): buckets with rows differ from the model"
        bits = _bits(c["values"])
        for b, w in want.items():
            if func == "count":
                assert int(bits[b]) == w["count"], f"{label} call {k}: count of bucket {b}"
                continue
            v = float(bits[b:b + 1].view(np.float64)[0]) if typ == L.TYPE_FLOAT else int(bits[b:b + 1].view(np.int64)[0])
            if func == "sum":
                ok = abs(v - w["sum"]) <= SUM_RTOL * abs(w["sum"]) if typ == L.TYPE_FLOAT else v == w["sum"]
                assert ok, f"{label} call {k}: sum of bucket {b} {v!r} vs {w['sum']!r}"
                continue
            t, wv = w[func]
            assert v == wv, f"{label} call {k} ({func}): bucket {b} {v!r} vs {wv!r}"
            if func in ("first", "last") or not multi:
                assert int(np.asarray(c["times"])[b]) == t, f"{label} call {k} ({func}): time of bucket {b}"


def _variants(case):
    """(name, expected path, AggQuery keywords, environment)"""
    il = case.default_path in (2, 3)
    return [("default", case.default_path, {}, None),
            ("strict", 2 if il else 1, dict(flags=L.Q_STRICT_ORDER), None),
            ("series", 2 if il else 1, dict(group="series"), None),
            ("map", 2 if il else 1, dict(group="map", series_group=np.arange(len(case.series)) % 3, n_groups=3), None),
            ("no_fast", 1, dict(flags=L.Q_NO_FAST), None),
            ("no_fused", 0, dict(flags=L.Q_NO_FUSED), None),
            ("where", 5, dict(filter=[KEEP]), None),
            ("where2", 4, dict(filter=[KEEP, KEEP2, "and"]), None),
            ("no_cols", 4, dict(filter=[KEEP]), "OGPU_NO_COLS")]


def run_path(g, case, calls, variant, monkeypatch, label, model=None, tmin=None, tmax=None, offset=None, interval=None, extra_flags=0,
             with_oracle=True):
    name, path, kw, env = variant
    kw = dict(kw)
    kw["flags"] = kw.get("flags", 0) | extra_flags
    tmin = case.tmin if tmin is None else tmin
    tmax = case.tmax if tmax is None else tmax
    label = f"{label} [{name}]"
    if path == 5 and max(Counter(c for _f, c in calls).values()) > OG_COLS_MAXMINE:
        path = 4  # k_fused_cols takes at most OG_COLS_MAXMINE calls per column
    if env:
        monkeypatch.setenv(env, "1")
    try:
        q = AggQuery(g.sh, calls, case.interval if interval is None else interval, tmin, tmax,
                     offset=case.offset if offset is None else offset, **kw).run()
    finally:
        if env:
            monkeypatch.delenv(env)
    st = q.stats()
    assert st["path"] == path, f"{label}: ran on path {st['path']}, expected {path}"
    gpu = q.dense_host()
    if with_oracle:
        ref = oracle.scan(g.sd, q.desc, threads=1)
        strict = bool(kw["flags"] & L.Q_STRICT_ORDER)
        compare_dense(gpu, ref, calls, len(calls) > 1, label, float_sum_exact=strict)
        if strict:
            assert st["rows_decoded"] == ref["rows_decoded"], label
    if model is not None and kw.get("group", "all") == "all":
        check_model(gpu, *model, g, calls, label)
    q.close()
    return st


CALL_SETS = [[(f, 0) for f in ALL6], [("sum", 0), ("count", 0), ("max", 0)], [("min", 1)], [("last", 0)]]


@pytest.mark.parametrize("name", list(CASES))
def test_time_grid(shards, monkeypatch, name):
    case = CASES[name]
    g = _shard(shards, name)
    model = _model(g, case)
    for calls in CALL_SETS:
        for v in _variants(case):
            run_path(g, case, calls, v, monkeypatch, f"{name} ({case.target}) {calls}", model)
    if case.stats:
        st = run_path(g, case, [("sum", 0), ("count", 0), ("max", 0)], _variants(case)[0], monkeypatch, name, model)
        for k, want in case.stats.items():
            assert st[k] == want, f"{name}: og_stats.{k} = {st[k]}, expected {want}"


def test_dt_2_40_eligibility(shards, monkeypatch):
    """k_fused_il takes a const-delta segment only when dt < 2^40: the odd series (dt = 2^40) go to the general kernel."""
    name = "cadence_2^40_edge"
    case, g = CASES[name], _shard(shards, name)
    st = run_path(g, case, [("sum", 0), ("count", 0)], _variants(case)[1], monkeypatch, name, _model(g, case))
    n_general = sum(1 for _t0, dt, _n in case.series if dt >= 1 << 40)
    assert st["il_state"] == 1 and st["general_segments"] == n_general, st


@pytest.mark.parametrize("name", ["cadence_7ns", "cadence_90s_windows_60s", "near_minus_2^62_7ns"])
def test_every_call_alone(shards, monkeypatch, name):
    """All six aggregates as single calls (selectors carry the row time) on every path."""
    case, g = CASES[name], _shard(shards, name)
    model = _model(g, case)
    for f in ALL6:
        for col in DISTINCT:
            for v in _variants(case):
                run_path(g, case, [(f, col)], v, monkeypatch, f"{name} {f}({COLS[col][0]})", model)


@pytest.mark.parametrize("name", ["cadence_7ns", "cadence_90s_windows_60s", "interval_dt_plus_1"])
def test_int_bool_and_null_columns(shards, monkeypatch, name):
    """Int and bool columns (path 1, and 0/4/5) and float, int and bool columns with nulls, single and multi."""
    case, g = CASES[name], _shard(shards, name)
    model = _model(g, case)
    paths = [("default", 1, {}, None), ("strict", 1, dict(flags=L.Q_STRICT_ORDER), None), ("no_fused", 0, dict(flags=L.Q_NO_FUSED), None),
             ("where", 5, dict(filter=[KEEP]), None), ("where2", 4, dict(filter=[KEEP, KEEP2, "and"]), None)]
    for col in (2, 3, 4, 5, 6):
        funcs = ["count", "first", "last", "min", "max"] + (["sum"] if COLS[col][1] != L.TYPE_BOOL else [])
        sets = [[(f, col)] for f in funcs] + [[(f, col) for f in funcs]]
        for calls in sets:
            for v in paths:
                if col == 2 and v[0] in ("default", "strict"):
                    v = (v[0], 1, v[2], v[3])  # a float column whose pages all carry nulls: k_fused_il takes none of them
                # single-call sum over a column with nulls, with a WHERE on another column: the reference places the window's
                # partial by a value index used as a row index (DESIGN.md "Deviations"), so only the model is compared
                quirk = calls == [("sum", col)] and col in NULL_EVERY and "filter" in v[2]
                run_path(g, case, calls, v, monkeypatch, f"{name} {calls}", model, with_oracle=not quirk)


def test_descending_records(shards):
    """ascending=False: og_query_next emits the same windows, latest first."""
    name = "cadence_7ns"
    case, g = CASES[name], _shard(shards, name)
    calls = [("sum", 0), ("min", 0), ("first", 1), ("count", 2)]

    def rows(asc):
        q = AggQuery(g.sh, calls, case.interval, case.tmin, case.tmax, offset=case.offset, ascending=asc).run()
        recs = list(q.records())
        assert q.stats()["path"] == 5
        q.close()
        times = np.concatenate([r["times"] for r in recs])
        cols = [(np.concatenate([r["cols"][k]["valid"] for r in recs]), np.concatenate([r["cols"][k]["values"] for r in recs]))
                for k in range(len(calls))]
        return times, cols

    ta, ca = rows(True)
    td, cd = rows(False)
    assert ta.size > 100 and np.array_equal(td, ta[::-1])
    for k, ((va, xa), (vd, xd)) in enumerate(zip(ca, cd)):
        assert np.array_equal(vd, va[::-1]), f"call {k}: validity"
        if calls[k][0] == "sum":
            assert np.allclose(xd, xa[::-1], rtol=SUM_RTOL, atol=0), f"call {k}: sums"
        else:
            assert np.array_equal(xd.view(np.uint64) if xd.dtype == np.float64 else xd, (xa.view(np.uint64) if xa.dtype == np.float64 else xa)[::-1]), f"call {k}"
    # one row per bucket that holds rows
    assert ta.size == len(_model(g, case)[1])


def test_query_grid_unaligned_range(shards, monkeypatch):
    """OG_Q_QUERY_GRID: the grid comes from the query range, not from the rows; tmin/tmax off every boundary and row."""
    name = "cadence_7ns"
    case, g = CASES[name], _shard(shards, name)
    tmin, tmax = T0 + 1236, T0 + 9805
    grid = tg.grid(case.interval, case.offset, tmin, tmax, g.tmin, g.tmax, query_grid=True)
    model = (grid, tg.bucket_rows(g.times, grid, case.interval, case.offset))
    for calls in ([(f, 0) for f in ALL6], [("sum", 0), ("count", 0), ("max", 0)], [("min", 1)]):
        for flags, path in ((L.Q_QUERY_GRID, 3), (L.Q_QUERY_GRID | L.Q_STRICT_ORDER, 2)):
            q = AggQuery(g.sh, calls, case.interval, tmin, tmax, offset=case.offset, flags=flags).run()
            assert q.stats()["path"] == path
            check_model(q.dense_host(), *model, g, calls, f"query grid {calls} flags={flags}")
            q.close()


def test_chunked_plan(shards, monkeypatch):
    """OGPU_CHUNK_SERIES=32: 40 series in two chunks, the second one a partial lane group."""
    monkeypatch.setenv("OGPU_CHUNK_SERIES", "32")
    for name in ("cadence_7ns", "interval_dt_plus_1", "fold_25_windows"):
        case, g = CASES[name], _shard(shards, name)
        model = _model(g, case)
        for calls in CALL_SETS:
            for v in _variants(case)[:2] + _variants(case)[4:7]:
                run_path(g, case, calls, v, monkeypatch, f"chunks {name} {calls}", model)


@pytest.mark.parametrize("which", ["max", "min"])
def test_clamped_grid_is_refused(which, monkeypatch):
    """Rows within one interval of MAX_TIME (MIN_TIME): Window() clamps the last (first) window, the reference's grid loses
    (misplaces) rows, and og_query_create refuses the query with OG_E_UNSUPPORTED (DESIGN.md "Deviations").  Without an
    interval, or with a range that stops short of the clamped window, the same rows are served."""
    t0 = tg.MAX_TIME - 7 * 299 if which == "max" else tg.MIN_TIME + 3
    case = Case("clamped", _n(t0, 7, 300), 100)
    g = GShard(case)
    try:
        grid = tg.grid(100, 0, *OPEN, g.tmin, g.tmax)
        assert grid.clamped
        for iv, off in ((100, 0), (100, 37), (7, 0)):
            with pytest.raises(L.OgpuError) as e:
                AggQuery(g.sh, [("count", 0)], iv, *OPEN, offset=off)
            assert e.value.status == L.OG_E_UNSUPPORTED, (iv, off)
        bounded = (OPEN[0], tg.MAX_TIME - 200) if which == "max" else (tg.MIN_TIME + 200, OPEN[1])
        for iv, (tmin, tmax) in ((0, OPEN), (100, bounded)):
            c = Case("served", case.series, iv, 0, tmin, tmax)
            model = _model(g, c)
            for calls in ([(f, 0) for f in ALL6], [("sum", 0), ("count", 0), ("max", 0)]):
                for v in _variants(c):
                    run_path(g, c, calls, v, monkeypatch, f"{which} limit iv={iv} {calls}", model)
    finally:
        g.sh.close()
