"""Shards of any segment geometry, built from per-series rows (test infrastructure).

openGemini writes segments of `max-rows-per-segment` rows (a setting, 1000 by default), so a valid TSSP file may hold segments of
1 to 2^32 - 1 rows, and a series may mix lengths (a merge rewrites spans of a longer-segment file into 1000-row segments).  This
module cuts the same per-series rows into whatever lengths a test names and encodes every page with the oracle's encoders:

    rows = series_rows(rng, n, KINDS, null_share)        # times + per column (values, valid), in numpy
    desc = shard_desc([rows, ...], types_of(KINDS), [[1000, 65537], ...])   # host L.ShardDesc (no device needed)
    sh, desc = open_shard(...)                           # the same, opened on the device

`window_model` is the plain numpy answer of a query over those rows (count, integer sum, min / max / first / last with their
times, the float sum's exact value and error bound), which must not depend on how the rows are cut."""
import math

import numpy as np

import oracle
from opengemini_b200 import _lib as L
from opengemini_b200.cursor import Shard

T0, SEC = 1_700_000_000_000_000_000, 1_000_000_000

# value kinds: the page form a long segment of each comes out as
KIND_TYPE = {"f_hi": L.TYPE_FLOAT,    # Gorilla, high entropy (G-hi)
             "f_lo": L.TYPE_FLOAT,    # Gorilla, few mantissa bits, runs of repeated values (G-lo)
             "f_raw": L.TYPE_FLOAT,   # incompressible bits: raw pages
             "i_s8b": L.TYPE_INT,     # random walk: Simple8b
             "i_const": L.TYPE_INT,   # one delta: const pages
             "i_wide": L.TYPE_INT,    # 58-bit values: raw pages for segments below three rows
             "bool": L.TYPE_BOOL}


def types_of(kinds):
    return [KIND_TYPE[k] for k in kinds]


def values(kind, rng, n):
    if kind == "f_hi":  # 36 random mantissa bits: 53 would make long pages raw (Gorilla above 90 % of raw)
        return 100.0 + np.floor(rng.random(n) * 2.0**36) / 2.0**36
    if kind == "f_lo":
        return np.repeat(20.0 + np.cumsum(rng.integers(-2, 3, (n + 3) // 4)) / 3.0, 4)[:n]
    if kind == "f_raw":  # as tests/test_gpu_parity._ragged_shard: random bits below 2^62 are finite, positive doubles below 2
        return rng.integers(0, 2**62, n).astype(np.uint64).view(np.float64)
    if kind == "i_s8b":
        return np.cumsum(rng.integers(-1000, 1001, n)).astype(np.int64)
    if kind == "i_const":
        return (7 + 3 * np.arange(n)).astype(np.int64)
    if kind == "i_wide":
        return rng.integers(-(1 << 57), 1 << 57, n).astype(np.int64)
    if kind == "bool":
        return rng.integers(0, 2, n).astype(np.uint8)
    raise KeyError(kind)


def series_rows(rng, n, kinds, null_share=0.0, t0=T0, irregular=False):
    """n rows of one series: {"times": int64[n], "cols": [(values, valid)] in the order of kinds}.  Times are 1 s apart, or
    1..89 s apart (Simple8b time pages) when irregular.  null_share: a float for every column, or one per column."""
    if irregular:
        t = t0 + np.concatenate([[0], np.cumsum(rng.integers(1, 90, n - 1))]).astype(np.int64) * SEC
    else:
        t = t0 + np.arange(n, dtype=np.int64) * SEC
    shares = null_share if isinstance(null_share, (list, tuple)) else [null_share] * len(kinds)
    cols = []
    for k, p in zip(kinds, shares):
        valid = np.ones(n, bool) if p == 0 else rng.random(n) >= p
        cols.append((values(k, rng, n), valid))
    return dict(times=t.astype(np.int64), cols=cols)


def _cuts(lengths, n):
    assert all(x > 0 for x in lengths) and sum(lengths) == n, (lengths, n)
    c = np.concatenate([[0], np.cumsum(lengths)]).astype(np.int64)
    return list(zip(c[:-1].tolist(), c[1:].tolist()))


def pages_of(rows, types, a, b):
    """[field pages of rows a:b], time page: the oracle's encoders; a column without nulls there gets a Full header"""
    out = []
    for (v, ok), ty in zip(rows["cols"], types):
        seg_ok = ok[a:b]
        out.append(oracle.field_page_encode(ty, np.ascontiguousarray(v[a:b]), None if seg_ok.all() else seg_ok.astype(np.uint8)))
    return out, oracle.time_page_encode(np.ascontiguousarray(rows["times"][a:b]))


def shard_desc(series, types, lengths, sids=None):
    """series: [series_rows(...)]; lengths: per series, the row count of each of its segments (summing to its rows).
    Returns an L.ShardDesc over host memory, pages laid out series-major, columns interleaved per segment."""
    nc = len(types)
    blob, pos = [], 0
    po = [[] for _ in range(nc)]; pl = [[] for _ in range(nc)]
    tpo, tpl, tmin, tmax, ssb = [], [], [], [], [0]

    def put(p):
        nonlocal pos
        blob.append(np.asarray(p, np.uint8)); off = pos; pos += len(p)
        return off, len(p)

    for rows, lens in zip(series, lengths):
        for a, b in _cuts(lens, rows["times"].size):
            fields, tp = pages_of(rows, types, a, b)
            for c, p in enumerate(fields):
                o, n = put(p); po[c].append(o); pl[c].append(n)
            o, n = put(tp); tpo.append(o); tpl.append(n)
            tmin.append(int(rows["times"][a])); tmax.append(int(rows["times"][b - 1]))
        ssb.append(len(tmin))
    sids = np.arange(1, len(series) + 1) if sids is None else sids
    return Shard.desc(np.concatenate(blob), sids, ssb, tmin, tmax, [(f"c{c}", types[c], po[c], pl[c]) for c in range(nc)], tpo, tpl)


def open_shard(series, types, lengths, sids=None):
    """(Shard on the device, its host L.ShardDesc for oracle.scan)"""
    d = shard_desc(series, types, lengths, sids)
    return Shard.open_desc(d, keepalive=d), d


def mixed(pattern, n):
    """segment lengths that repeat `pattern` and end with whatever is left"""
    out, left, i = [], n, 0
    while left:
        x = min(left, pattern[i % len(pattern)])
        out.append(x); left -= x; i += 1
    return out


# ---------------------------------------------------------------------------------------------------------------
# the numpy window model
# ---------------------------------------------------------------------------------------------------------------
def grid(interval, offset, tmin, tmax):
    """(start, n_buckets) of the dense record: windows of `interval` ns aligned to `offset`, from the one holding tmin to the one
    holding tmax; one bucket starting at 0 without an interval"""
    if interval == 0:
        return 0, 1
    start = tmin - (tmin - offset) % interval
    return start, (tmax - start) // interval + 1


def window_model(series, col, typ, interval, offset, tmin, tmax, groups):
    """Per (group, window) over the valid rows of column `col` in [tmin, tmax]: count, integer sum (wrapping), min / max with the
    earliest time among equal extremes, first / last with the larger value among equal times, and for floats the exact sum
    (math.fsum) and sum of |x|.  groups: the group of each series.  Returns {name: array over n_groups * n_buckets}, "valid"."""
    start, nb = grid(interval, offset, tmin, tmax)
    ng = int(max(groups)) + 1
    cells = ng * nb
    t_all, v_all, cell_all = [], [], []
    for rows, g in zip(series, groups):
        t = rows["times"]
        v, ok = rows["cols"][col]
        m = ok & (t >= tmin) & (t <= tmax)
        b = (t[m] - start) // interval if interval else np.zeros(int(m.sum()), np.int64)
        t_all.append(t[m]); v_all.append(v[m]); cell_all.append(g * nb + b)
    t, v, cell = np.concatenate(t_all), np.concatenate(v_all), np.concatenate(cell_all).astype(np.int64)
    count = np.bincount(cell, minlength=cells).astype(np.int64)
    out = dict(valid=count > 0, count=count, n_buckets=nb, start=start)
    key = v.astype(np.float64) if typ == L.TYPE_FLOAT else v.astype(np.int64)
    if typ == L.TYPE_INT:
        s = np.zeros(cells, np.int64)
        np.add.at(s, cell, v.astype(np.int64))  # wraps like the reference's int64 sum
        out["sum"] = s
    order_min = np.lexsort((t, key, cell))          # by cell, then value ascending, then time ascending
    order_max = np.lexsort((t, -key, cell))
    order_first = np.lexsort((-key, t, cell))       # earliest time, larger value on equal times
    order_last = np.lexsort((-key, -t, cell))
    for name, order in (("min", order_min), ("max", order_max), ("first", order_first), ("last", order_last)):
        c = cell[order]
        head = np.ones(c.size, bool)
        head[1:] = c[1:] != c[:-1]
        pick = order[head]
        val = np.zeros(cells, v.dtype); tim = np.zeros(cells, np.int64)
        val[cell[pick]] = v[pick]; tim[cell[pick]] = t[pick]
        out[name], out[name + "_time"] = val, tim
    if typ == L.TYPE_FLOAT:
        exact, mag = np.zeros(cells), np.zeros(cells)
        order = np.argsort(cell, kind="stable")
        c, vs = cell[order], v[order]
        bounds = np.flatnonzero(np.r_[True, c[1:] != c[:-1], True])
        for a, b in zip(bounds[:-1], bounds[1:]):
            exact[c[a]] = math.fsum(vs[a:b].tolist())
            mag[c[a]] = math.fsum(np.abs(vs[a:b]).tolist())
        out["sum_exact"], out["sum_abs"] = exact, mag
    return out


def check_against_model(dense, calls, model, typ, label, multi=None):
    """dense: AggQuery.dense_host() / oracle.scan() of `calls` over one column; every cell against window_model.  Float sums lie
    within n * 2^-53 * sum|x| of the exact sum of the window's rows (n: the window's row count)."""
    assert dense["n_buckets"] == model["n_buckets"] and dense["start"] == model["start"], label
    ok = model["valid"]
    multi = len(calls) > 1 if multi is None else multi  # several calls: min / max carry no time
    for k, (f, _c) in enumerate(calls):
        col = dense["cols"][k]
        assert np.array_equal(np.asarray(col["valid"]).astype(bool), ok), f"{label} {f}: validity"
        got = np.asarray(col["values"])
        if f == "count":
            assert np.array_equal(got.view(np.int64)[ok], model["count"][ok]), f"{label} count"
            continue
        if f == "sum" and typ == L.TYPE_FLOAT:
            g = got.view(np.float64)[ok]
            bound = model["count"][ok] * 2.0**-53 * model["sum_abs"][ok]
            err = np.abs(g - model["sum_exact"][ok])
            assert np.all(err <= bound), f"{label} sum: off by {float((err - bound).max()):.3e} beyond n*2^-53*sum|x|"
            continue
        want = model[f][ok]
        if typ == L.TYPE_BOOL:
            assert np.array_equal(got.view(np.uint64)[ok] != 0, want != 0), f"{label} {f}"
        else:
            assert np.array_equal(got.view(np.uint64)[ok], want.view(np.uint64)), f"{label} {f}"
        if f in ("first", "last") or (f in ("min", "max") and not multi):
            assert np.array_equal(np.asarray(col["times"])[ok], model[f + "_time"][ok]), f"{label} {f} times"
