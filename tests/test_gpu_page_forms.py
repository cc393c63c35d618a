"""Every decode and aggregate kernel on the page forms of tests/page_forms.py, against the oracle.

Each aggregate case states the path it means to take and asserts it from og_stats, so a planner change cannot route around it:
  3 / 2  k_fused_il, folded / per-series (strict order): one float column whose pages are Gorilla or raw with a Full header
  1      the pull-iterator kernel (k_fused_segment): any single column (Q_NO_FAST, or int / bool / other float codecs)
  0      the tile path: Q_NO_FUSED
  5      k_fused_cols: two columns or one WHERE term, const-delta time pages, segments of <= 1024 rows
  4      k_fused_multi: the same with OGPU_NO_COLS=1, or a Simple8b / raw time page, or a longer segment
Everything is bitwise against the oracle except float sums on path 3 (SUM_RTOL, test_gpu_parity's rule)."""
import ctypes as C

import numpy as np
import pytest

import oracle
import page_forms as pf
from opengemini_b200 import AggQuery, Shard
from opengemini_b200 import _lib as L
from test_gpu_parity import compare_dense, run_both

pytestmark = pytest.mark.gpu

T0, SEC = pf.T0, pf.SEC
ALL6 = ["count", "sum", "min", "max", "first", "last"]
VALUES = pf.value_entries()
TIMES = pf.time_entries()
BY_NAME = {e.name: e for e in VALUES + TIMES}


@pytest.fixture(scope="module", autouse=True)
def _device():
    Shard.init(0)


def _open(series, types):
    """series: list of series, each a list of segments (times, [page of each column]); one shard, every column of type types[c]"""
    nc = len(types)
    blob, pos = [], 0
    po = [[] for _ in range(nc)]; pl = [[] for _ in range(nc)]
    tpo, tpl, tmin, tmax, ssb = [], [], [], [], [0]

    def put(p):
        nonlocal pos
        blob.append(np.asarray(p, np.uint8)); off = pos; pos += len(p)
        return off, len(p)
    for segs in series:
        for t, pages in segs:
            for c in range(nc):
                o, n = put(pages[c]); po[c].append(o); pl[c].append(n)
            o, n = put(oracle.time_page_encode(np.asarray(t, np.int64)))
            tpo.append(o); tpl.append(n); tmin.append(int(t[0])); tmax.append(int(t[-1]))
        ssb.append(len(tmin))
    sh = Shard.open(np.concatenate(blob), np.arange(1, len(series) + 1), ssb, tmin, tmax,
                    [(f"c{c}", types[c], po[c], pl[c]) for c in range(nc)], tpo, tpl)
    return sh, oracle.shard_desc_from_export(sh.export())


def _fpages(vals):
    return [oracle.field_page_encode(L.TYPE_FLOAT, np.asarray(v, np.float64)) for v in vals]


def _zeros_unsigned(d):
    """-0.0 cells as +0.0 (values only: validity and times stay as they are)"""
    for c in d["cols"]:
        u = np.asarray(c["values"]).view(np.uint64).copy()
        u[u == np.uint64(1 << 63)] = 0
        c["values"] = u
    return d


def _query(sh, sd, calls, iv, tmin, tmax, path, flags, monkeypatch, label, zeros_as_floats=False, **kw):
    """run the query the way `path` names, assert the path, compare with the oracle (zeros_as_floats: +0.0 == -0.0)"""
    with monkeypatch.context() as m:
        if path == 4:  # harmless where the shard's time pages already rule k_fused_cols out
            m.setenv("OGPU_NO_COLS", "1")
        q = AggQuery(sh, calls, iv, tmin, tmax, flags=flags, **kw).run()
        try:
            st = q.stats()
            assert st["path"] == path, f"{label}: path {st['path']}, wanted {path}"
            if path in (2, 3):
                assert st["il_state"] == 1, label
            if path == 3 and (iv == 0 or iv >= 60 * SEC):  # short windows may take lanes out of step (og_stats)
                assert st["per_series_cells_used"] == 0, label
            gpu = q.dense_host()
            ref = oracle.scan(sd, q.desc, threads=1)
        finally:
            q.close()
    if zeros_as_floats:
        gpu, ref = _zeros_unsigned(gpu), _zeros_unsigned(ref)
    compare_dense(gpu, ref, calls, len(calls) > 1, f"{label} [path {path}]", float_sum_exact=path != 3)
    return gpu, ref


def _il_eligible(e):
    return e.typ == L.TYPE_FLOAT and pf.read_header(e.page)["kind"] == "full" and pf.codec_of(e.typ, e.page) in ("gorilla", "raw")


def _single_paths(e):
    """(flags, path) of the single-column paths that can serve the entry"""
    out = []
    if _il_eligible(e):
        if "nan" not in e.tags:  # the folded order makes no promise with NaN partials (DESIGN.md "Exactness")
            out.append((0, 3))
        out += [(L.Q_STRICT_ORDER, 2), (L.Q_STRICT_ORDER | L.Q_NO_FAST, 1)]
    else:
        out.append((L.Q_STRICT_ORDER, 1))
    out.append((L.Q_STRICT_ORDER | L.Q_NO_FUSED, 0))
    return out


def _multi_paths(rows, const_time=True):
    return ([5] if rows <= 1024 and const_time else []) + [4]


def _funcs(typ):
    return ALL6 if typ != L.TYPE_BOOL else ["count", "min", "max", "first", "last"]


# ---------------------------------------------------------------------------------------------------------------
# decode
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", [e.name for e in VALUES + TIMES])
def test_decode_segment(name):
    e = BY_NAME[name]
    if e.typ == pf.TIME:
        typ, page, times = L.TYPE_FLOAT, _fpages([100 + np.arange(e.rows) * 0.001 + np.random.default_rng(1).random(e.rows)])[0], e.cells
    else:
        typ, page, times = e.typ, e.page, e.times()
    sh, _sd = _open([[(times, [page])]], [typ])
    want_v, want_ok = oracle.field_page_decode(typ, page, cap=times.size + 8)
    want_t = oracle.time_page_decode(e.page if e.typ == pf.TIME else oracle.time_page_encode(times), cap=times.size + 8)
    for desc in (False, True):
        rec = sh.decode_segment(0, descending=desc)
        r = (lambda a: np.ascontiguousarray(a[::-1])) if desc else (lambda a: a)
        assert np.array_equal(rec["times"], r(want_t)), (name, desc)
        col = rec["cols"][0]
        assert np.array_equal(col["valid"], r(want_ok)), (name, desc)
        assert col["nil_count"] == int((~want_ok).sum())
        w = r(want_v)
        assert np.array_equal(col["values"].view(np.uint8), w.view(np.uint8)), (name, desc)
    sh.close()


# ---------------------------------------------------------------------------------------------------------------
# aggregates: every entry, every path that can serve it, single-call and multi-call
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", [e.name for e in VALUES])
def test_aggregates_on_every_path(name, monkeypatch):
    e = BY_NAME[name]
    t = e.times()
    sh, sd = _open([[(t, [e.page, e.page])]], [e.typ, e.typ])
    tmin, tmax = int(t[0]), int(t[-1])
    funcs = _funcs(e.typ)
    for flags, path in _single_paths(e):
        for f in funcs:
            _query(sh, sd, [(f, 0)], 60 * SEC, tmin, tmax, path, flags, monkeypatch, f"{name} {f}")
        for iv in (7 * SEC, 0):
            _query(sh, sd, [(f, 0) for f in funcs], iv, tmin, tmax, path, flags, monkeypatch, f"{name} multi iv={iv}")
        if e.rows > 30:
            _query(sh, sd, [("max", 0), ("sum" if e.typ != L.TYPE_BOOL else "count", 0)], 60 * SEC, tmin + 17 * SEC + 3, tmax - 5 * SEC,
                   path, flags, monkeypatch, f"{name} mid-range")
    simple = [("sum", 0), ("count", 0), ("count", 1), ("sum", 1)] if e.typ != L.TYPE_BOOL else [("count", 0), ("count", 1)]
    for path in _multi_paths(e.rows, pf.time_codec(oracle.time_page_encode(t)) in ("t_const", "t_one")):  # 2 rows: a raw time page
        two = [(f, 0) for f in funcs[:3]] + [(f, 1) for f in funcs[3:]]
        for iv in (60 * SEC, 0):
            _query(sh, sd, two, iv, tmin, tmax, path, L.Q_STRICT_ORDER, monkeypatch, f"{name} two columns iv={iv}")
            _query(sh, sd, simple, iv, tmin, tmax, path, L.Q_STRICT_ORDER, monkeypatch, f"{name} two columns count/sum iv={iv}")
        if e.rows > 200:
            _query(sh, sd, two, 45 * SEC, tmin + 123 * SEC + 1, tmax, path, L.Q_STRICT_ORDER, monkeypatch, f"{name} two columns mid-range")
    sh.close()


# ---------------------------------------------------------------------------------------------------------------
# lane groups built to stress k_fused_il
# ---------------------------------------------------------------------------------------------------------------
LANE_FORMS = {"dense": dict(codec="gorilla", leads_within={0}, min_run66=700), "zeros": dict(codec="gorilla", min_zero_frac=0.99),
              "lead2": dict(codec="gorilla", leads={2}, leads_within={2}), "switch": dict(codec="gorilla", leads={0, 2}, min_lead_switches=10)}


def _lane_shard(kinds, seed, n_seg=2):
    rng = np.random.default_rng(seed)
    series = []
    for k in kinds:
        segs = []
        for g in range(n_seg):
            v = pf.lane_values(k, rng)
            t = T0 + (np.arange(1000, dtype=np.int64) + g * 1000) * SEC
            page = _fpages([v])
            if k in LANE_FORMS:  # every lane holds the form it stands for
                e = pf.Entry(f"lane {k}", L.TYPE_FLOAT, v, np.ones(v.size, bool), page[0], LANE_FORMS[k])
                assert not pf.check_forms(e)
            segs.append((t, page))
        series.append(segs)
    return _open(series, [L.TYPE_FLOAT])


@pytest.mark.parametrize("mix", ["dense_and_zeros", "lead2", "switch"])
def test_lane_groups(mix, monkeypatch):
    """32-series lane groups (and a partial 33rd..40th): lanes whose streams differ by 65 bits per row drift far beyond the
    64-row ring; lanes all at leading count 2 sit on the fast path's edge; lanes switch between leading count 2 and 0/1"""
    kinds = {"dense_and_zeros": ["dense" if s % 3 else "zeros" for s in range(40)], "lead2": ["lead2"] * 40,
             "switch": ["switch" if s % 2 else "lead2" for s in range(40)]}[mix]
    sh, sd = _lane_shard(kinds, seed=len(mix))
    tmax = T0 + 1999 * SEC
    for calls in ([(f, 0) for f in ALL6], [("sum", 0), ("count", 0), ("max", 0)], [("min", 0)], [("first", 0), ("last", 0)]):
        for iv in (60 * SEC, 7 * SEC):
            _query(sh, sd, calls, iv, T0, tmax, 3, 0, monkeypatch, f"{mix} {calls} iv={iv}")
            _query(sh, sd, calls, iv, T0, tmax, 2, L.Q_STRICT_ORDER, monkeypatch, f"{mix} {calls} iv={iv}")
    run_both(sh, sd, [("sum", 0), ("max", 0)], 45 * SEC, T0 + 777 * SEC, T0 + 1500 * SEC, f"{mix} mid-range")
    run_both(sh, sd, [("last", 0)], 60 * SEC, T0, tmax, f"{mix} per series", group="series")
    sh.close()


# ---------------------------------------------------------------------------------------------------------------
# WHERE
# ---------------------------------------------------------------------------------------------------------------
WHERE_NAMES = ["g_sign", "g_wrap", "g_special_pinf", "f_raw", "f_raw_nan", "f_same", "f_same0_nulls", "f_rle_nulls_bmoff4", "f_one", "f_empty",
               "i_const_neg", "i_s8b_all_nulls_bmoff2", "i_raw", "i_s8b_hi", "i_one", "i_empty", "b_full_nulls_bmoff3", "b_full", "b_one", "b_empty"]


@pytest.mark.parametrize("name", WHERE_NAMES)
def test_where_on_each_codec(name, monkeypatch):
    """one term on a column of each codec (the filter column is the value column's page, so every row meets its own value);
    NaN rows of a raw page under every operator (ordered compares pass NaN, = fails it)"""
    e = BY_NAME[name]
    t = e.times()
    sh, sd = _open([[(t, [e.page, e.page])]], [e.typ, e.typ])
    v = e.cells[e.valid]
    if e.typ == L.TYPE_FLOAT:
        fin = v[np.isfinite(v)]
        consts = [float(np.median(fin)) if fin.size else 0.5, 0.0]
    elif e.typ == L.TYPE_INT:
        consts = [int(np.median(v)) if v.size else 0, 0]
    else:
        consts = [1, 0]
    ops = ["<", "<=", ">", ">=", "=", "!="] if "nan" in e.tags or e.typ == L.TYPE_BOOL else [">", "=", "!="]
    calls = [("count", 0), ("sum" if e.typ != L.TYPE_BOOL else "count", 0), ("max", 0), ("first", 0)]
    for c in consts:
        for op in ops:
            flt = [("term", 1, op, c)]
            for path, flags in ((5, L.Q_STRICT_ORDER), (4, L.Q_STRICT_ORDER), (0, L.Q_STRICT_ORDER | L.Q_NO_FUSED)):
                if path == 5 and e.rows > 1024:
                    continue
                _query(sh, sd, calls, 60 * SEC, int(t[0]), int(t[-1]), path, flags, monkeypatch, f"{name} where {op} {c}", filter=flt)
    sh.close()


def test_int_column_against_a_float_constant_next_to_2_pow_53(monkeypatch):
    """Int64ToFloat64Slice: the int column is compared as doubles, so 2^53 + 1 equals 2^53 + 0.0"""
    e = BY_NAME["i_near53"]
    t = e.times()
    sh, sd = _open([[(t, [e.page, e.page])]], [L.TYPE_INT, L.TYPE_INT])
    for c in (float(2**53), float(2**53 + 2), float(2**53) - 1.0, 9007199254740993.0):
        for op in ("<", "<=", ">", ">=", "=", "!="):
            for path, flags in ((5, 0), (4, 0), (0, L.Q_NO_FUSED)):
                _query(sh, sd, [("count", 0), ("sum", 0), ("min", 0)], 60 * SEC, int(t[0]), int(t[-1]), path, flags | L.Q_STRICT_ORDER,
                       monkeypatch, f"2^53 {op} {c!r}", filter=[("term", 1, op, c)])
    sh.close()


# ---------------------------------------------------------------------------------------------------------------
# value extremes and signed zeros
# ---------------------------------------------------------------------------------------------------------------
def _canon_nan(d):
    """every NaN as one bit pattern (float columns only in the query below)"""
    for c in d["cols"]:
        u = np.asarray(c["values"]).view(np.uint64).copy()
        u[np.isnan(u.view(np.float64))] = 0x7FF8000000000000
        c["values"] = u
    return d


def test_infinities_in_two_segments_of_one_window_and_sums_that_overflow():
    """+Inf in one segment and -Inf in the next: the window's sum is NaN in the reference too (the NaN's bits are not compared:
    x86 and the GPU write different default NaNs for Inf - Inf); sums of DBL_MAX-sized values overflow to +-Inf"""
    pinf, ninf = BY_NAME["g_special_pinf"].cells, BY_NAME["g_special_ninf"].cells
    big = np.full(1000, pf.DBL_MAX / 3)
    bigg = pf.DBL_MAX / 2 * (1 + np.random.default_rng(5).random(1000))
    series = [[(T0 + np.arange(1000, dtype=np.int64) * SEC, _fpages([pinf])), (T0 + np.arange(1000, 2000, dtype=np.int64) * SEC, _fpages([ninf]))],
              [(T0 + np.arange(1000, dtype=np.int64) * SEC, _fpages([big])), (T0 + np.arange(1000, 2000, dtype=np.int64) * SEC, _fpages([-bigg]))]]
    sh, sd = _open(series, [L.TYPE_FLOAT])
    for iv in (0, 3600 * SEC, 60 * SEC):
        for flags, path in ((L.Q_STRICT_ORDER, 2), (L.Q_STRICT_ORDER | L.Q_NO_FAST, 1), (L.Q_STRICT_ORDER | L.Q_NO_FUSED, 0)):
            for group in ("all", "series"):
                calls = [(f, 0) for f in ALL6]
                q = AggQuery(sh, calls, iv, T0, T0 + 1999 * SEC, flags=flags, group=group).run()
                assert q.stats()["path"] == path
                gpu = _canon_nan(q.dense_host())
                ref = _canon_nan(oracle.scan(sd, q.desc, threads=1))
                q.close()
                compare_dense(gpu, ref, calls, True, f"inf iv={iv} path {path} {group}")
                s = np.asarray(gpu["cols"][1]["values"]).view(np.float64)
                assert np.isnan(s).any() or iv != 0 or group != "all"
    sh.close()


def test_signed_zeros_at_the_same_rows_of_different_series(monkeypatch):
    """+0.0 in even series and -0.0 in odd series at the same rows, where they are each window's extreme, first and last value:
    the reference keeps the earlier series' zero on the tie.  The odd series are Gorilla pages of repeated values, the even ones
    raw pages, so the odd series have the shorter streams and k_fused_il's lane sort (key: domain, stream words; ascending)
    puts an odd series, a -0.0 one, into lane 0 of every group.  Every path is bitwise under the strict order; the folded order
    (path 3) may keep the other zero of a tie (DESIGN.md "Exactness"), so there the zeros compare as floats and everything
    else, times included, bitwise."""
    rng = np.random.default_rng(17)
    series, words = [], {0: [], 1: []}
    for s in range(40):
        z = 0.0 if s % 2 == 0 else -0.0
        pos = 1.0 + (rng.random(1000) if s % 2 == 0 else np.repeat(rng.random(250), 4))
        pos[::60] = z  # the first row of every 60 s window
        pos[30::60] = z
        neg = -(1.0 + (rng.random(1000) if s % 2 == 0 else np.repeat(rng.random(250), 4)))
        neg[::60] = z
        neg[59::60] = z
        pages = _fpages([pos, neg])
        for p in pages:
            h = pf.read_header(p)
            assert pf.codec_of(L.TYPE_FLOAT, p) == ("raw" if s % 2 == 0 else "gorilla"), s
            words[s % 2].append(2 * 1000 if s % 2 == 0 else (h["block"].size + 3) // 4)  # raw: 8 B a row; Gorilla: its bytes
        series.append([(T0 + np.arange(1000, dtype=np.int64) * SEC, pages)])
    assert max(words[1]) < min(words[0]) // 2  # with the stream pad of a few words, odd series still sort first
    sh, sd = _open(series, [L.TYPE_FLOAT, L.TYPE_FLOAT])
    # the two-column shard serves the single-column paths per column; values of column 0 sit >= 0, of column 1 <= 0
    for col, funcs in ((0, ["min", "first"]), (1, ["max", "first", "last"])):
        for f in funcs:
            for flags, path in ((0, 3), (L.Q_STRICT_ORDER, 2), (L.Q_STRICT_ORDER | L.Q_NO_FAST, 1), (L.Q_STRICT_ORDER | L.Q_NO_FUSED, 0)):
                _query(sh, sd, [(f, col)], 60 * SEC, T0, T0 + 999 * SEC, path, flags, monkeypatch, f"signed zero {f}(c{col})",
                       zeros_as_floats=path == 3)
    for path in (5, 4):
        _query(sh, sd, [("min", 0), ("first", 0), ("max", 1), ("last", 1)], 60 * SEC, T0, T0 + 999 * SEC, path, L.Q_STRICT_ORDER,
               monkeypatch, "signed zero two columns")
    sh.close()


# ---------------------------------------------------------------------------------------------------------------
# timestamps before 1970, across 0, in [-2^52, 0), and an open range
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["t_pre1970", "t_cross0", "t_nan_doubles", "t_pre1970_s8b"])
def test_negative_times(name, monkeypatch):
    """Three series on the same times, so selector ties fall on equal times.  Where those times lie in [-2^52, 0) the
    reference compares them as the doubles their bits spell, which are NaN: its answer then depends on the series order, so
    that entry runs under the strict order only."""
    e = BY_NAME[name]
    t = e.cells
    rng = np.random.default_rng(3)
    vals = [np.round(rng.random(t.size) * 4) / 4 + 100 + rng.random(t.size) * (rng.random(t.size) < 0.3) for _ in range(3)]
    sh, sd = _open([[(t, _fpages([v, v[::-1].copy()]))] for v in vals], [L.TYPE_FLOAT, L.TYPE_FLOAT])
    const = pf.time_codec(e.page) == "t_const"
    folded_ok = "nan_times" not in e.tags
    lo, hi = int(t[0]), int(t[-1])
    for iv, off in ((60 * SEC, 0), (7 * SEC, 3 * SEC), (3600 * SEC, -13 * SEC), (0, 0)):
        for f in ALL6:
            paths = [(L.Q_STRICT_ORDER | L.Q_NO_FAST, 1), (L.Q_STRICT_ORDER | L.Q_NO_FUSED, 0)]
            if const:  # k_fused_il takes const-delta time pages only
                paths += ([(0, 3)] if folded_ok else []) + [(L.Q_STRICT_ORDER, 2)]
            for flags, path in paths:
                _query(sh, sd, [(f, 0)], iv, lo + 5 * SEC + 1, hi - 2 * SEC, path, flags, monkeypatch, f"{name} {f} iv={iv} off={off}", offset=off)
        for path in _multi_paths(t.size, const):
            _query(sh, sd, [("first", 0), ("last", 0), ("min", 1), ("max", 1)], iv, lo, hi, path, L.Q_STRICT_ORDER, monkeypatch,
                   f"{name} two columns iv={iv}", offset=off)
    for iv in (0, 3600 * SEC):  # an open range
        _query(sh, sd, [(f, 0) for f in ALL6], iv, pf.I64_MIN, pf.I64_MAX, 2 if const else 1, L.Q_STRICT_ORDER, monkeypatch,
               f"{name} open range iv={iv}")
        _query(sh, sd, [("count", 0), ("first", 1)], iv, pf.I64_MIN, pf.I64_MAX, _multi_paths(t.size, const)[0], L.Q_STRICT_ORDER,
               monkeypatch, f"{name} open range two columns iv={iv}")
    sh.close()


# ---------------------------------------------------------------------------------------------------------------
# device encoders against the oracle's, byte for byte
# ---------------------------------------------------------------------------------------------------------------
ENC = [e.name for e in VALUES if e.encoder_built and e.rows <= 1000]


@pytest.mark.parametrize("name", ENC)
def test_device_encoder_writes_the_oracle_bytes(name):
    import torch
    e = BY_NAME[name]
    want = oracle.field_page_encode(e.typ, e.cells, None if e.valid.all() else e.valid.astype(np.uint8))
    assert np.array_equal(want, e.page)
    cells = torch.from_numpy(np.ascontiguousarray(e.cells)).cuda()
    valid = torch.from_numpy(e.valid.astype(np.uint8)).cuda()
    rows = torch.tensor([e.rows], dtype=torch.int32, device="cuda")
    out = torch.zeros(16384, dtype=torch.uint8, device="cuda")
    off = torch.zeros(1, dtype=torch.int64, device="cuda")
    ln = torch.zeros(1, dtype=torch.int32, device="cuda")
    total = C.c_uint64()
    L.check(L.lib().og_encode_pages(e.typ, 0, cells.data_ptr(), None if e.valid.all() else valid.data_ptr(), rows.data_ptr(), 1, 1000,
                                    out.data_ptr(), out.numel(), off.data_ptr(), ln.data_ptr(), C.byref(total)), "og_encode_pages")
    got = out.cpu().numpy()[int(off[0]):int(off[0]) + int(ln[0])]
    assert np.array_equal(got, want), f"{name}: device {got.size} B, oracle {want.size} B"


# ---------------------------------------------------------------------------------------------------------------
# merge at open: an out-of-order file of catalogue pages over an ordered file
# ---------------------------------------------------------------------------------------------------------------
def test_out_of_order_file_of_catalogue_pages():
    """The merge decodes the out-of-order file's pages (bitmaps at offsets 3..5, one-row, Empty, Same, RLE, const-delta int) and
    re-encodes the merged rows with og_encode_pages; the merged rows must equal the row-rule model of test_gpu_out_of_order"""
    from test_gpu_out_of_order import _check_rows, _file_desc, _model, _series
    rng = np.random.default_rng(23)
    n = 2000
    ordered = {}
    for sid in (1, 2):
        cols = {"bv": (L.TYPE_BOOL, (rng.random(n) < 0.5).astype(np.uint8), rng.random(n) > 0.05),
                "fv": (L.TYPE_FLOAT, 100 + rng.random(n), rng.random(n) > 0.05),
                "iv": (L.TYPE_INT, rng.integers(-50, 50, n).cumsum(), rng.random(n) > 0.05)}
        ordered[sid] = _series(T0 + np.arange(n, dtype=np.int64) * SEC, cols)
    # segments of the out-of-order series 1, one page per column (names sorted: bv, fv, iv), in time order
    segs = [(["b_full_nulls_bmoff3", "f_rle_nulls_bmoff4", "i_const_neg_nulls_bmoff5"], lambda r: T0 + np.arange(r, dtype=np.int64) * SEC),
            (["b_one", "f_one", "i_one"], lambda r: np.array([T0 + 1500 * SEC + SEC // 2], np.int64)),
            (["b_full", "f_same", "i_const_pos"], lambda r: T0 + (1600 + 2 * np.arange(r, dtype=np.int64)) * SEC),
            (["b_empty", "f_empty", "i_empty"], lambda r: T0 + (4000 + np.arange(r, dtype=np.int64)) * SEC)]
    blob, pos, po, pl, tpo, tpl, tmin, tmax = [], 0, [[], [], []], [[], [], []], [], [], [], []
    times, cells = [], {"bv": ([], []), "fv": ([], []), "iv": ([], [])}
    for names, tf in segs:
        es = [BY_NAME[x] for x in names]
        assert len({e.rows for e in es}) == 1, names
        t = tf(es[0].rows)
        for c, (col, e) in enumerate(zip(("bv", "fv", "iv"), es)):
            po[c].append(pos); pl[c].append(e.page.size); blob.append(e.page); pos += e.page.size
            cells[col][0].append(e.cells); cells[col][1].append(e.valid)
        tp = oracle.time_page_encode(t)
        tpo.append(pos); tpl.append(tp.size); blob.append(tp); pos += tp.size
        tmin.append(int(t[0])); tmax.append(int(t[-1])); times.append(t)
    ooo_desc = Shard.desc(np.concatenate(blob), [1], [0, len(segs)], tmin, tmax,
                          [(col, typ, po[c], pl[c]) for c, (col, typ) in enumerate((("bv", L.TYPE_BOOL), ("fv", L.TYPE_FLOAT), ("iv", L.TYPE_INT)))],
                          tpo, tpl)
    ooo = {1: _series(np.concatenate(times), {col: (typ, np.concatenate(cells[col][0]), np.concatenate(cells[col][1]))
                                              for col, typ in (("bv", L.TYPE_BOOL), ("fv", L.TYPE_FLOAT), ("iv", L.TYPE_INT))})}
    sh = Shard.open_files([(_file_desc(ordered), False), (ooo_desc, True)])
    assert sh.merge_info()["series_merged"] == 1
    _check_rows(sh, _model([(ordered, False), (ooo, True)]))
    sh.close()
