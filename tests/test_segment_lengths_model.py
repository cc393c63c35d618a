"""The segment-geometry builder and window model of tests/segment_shards.py, on the CPU.

The builder's pages decode back through the oracle to the rows it was given, at every segment length the GPU tests use; the
numpy window model agrees with oracle.scan on small shards cut at several lengths, so the GPU tests may hold the library to it."""
import numpy as np
import pytest

import oracle
import segment_shards as ss
from opengemini_b200 import _lib as L

SEC = ss.SEC
LENGTHS = [1, 2, 3, 31, 32, 33, 999, 1000, 1001, 1023, 1024, 1025, 2048, 4095, 4096, 8192, 65535, 65536, 65537]
KINDS = ["f_hi", "f_lo", "f_raw", "i_s8b", "i_const", "i_wide", "bool"]


def _codec(typ, page):
    """the value codec of a field page (header forms as tests/page_forms.py reads them)"""
    import page_forms as pf
    return pf.codec_of(typ, page)


@pytest.mark.parametrize("n", LENGTHS)
def test_pages_decode_back_to_the_rows(n):
    rng = np.random.default_rng(n)
    types = ss.types_of(KINDS)
    for irregular in (False, True):
        rows = ss.series_rows(rng, n, KINDS, [0, 0.1, 0, 0.3, 0, 0, 0.05], irregular=irregular)
        fields, tp = ss.pages_of(rows, types, 0, n)
        assert np.array_equal(oracle.time_page_decode(tp, cap=n + 8), rows["times"])
        for (v, ok), ty, page in zip(rows["cols"], types, fields):
            got, gok = oracle.field_page_decode(ty, page, cap=n + 8)
            assert np.array_equal(gok, ok)
            assert np.ascontiguousarray(got).tobytes() == np.ascontiguousarray(v[ok]).tobytes()


def test_long_pages_take_the_forms_they_stand_for():
    rng = np.random.default_rng(3)
    n = 65537
    rows = ss.series_rows(rng, n, KINDS)
    fields, tp = ss.pages_of(rows, ss.types_of(KINDS), 0, n)
    forms = [_codec(ty, p) for ty, p in zip(ss.types_of(KINDS), fields)]
    assert forms[:5] == ["gorilla", "gorilla", "raw", "s8b", "const"], forms
    import page_forms as pf
    assert pf.time_codec(tp) == "t_const"
    irregular = ss.series_rows(rng, n, ["f_hi"], irregular=True)
    assert pf.time_codec(ss.pages_of(irregular, [L.TYPE_FLOAT], 0, n)[1]) == "t_s8b"
    two = ss.series_rows(rng, 2, ["i_wide"])
    assert _codec(L.TYPE_INT, ss.pages_of(two, [L.TYPE_INT], 0, 2)[0][0]) == "raw"


def test_mixed_lengths():
    assert ss.mixed([1000, 65537], 70000) == [1000, 65537, 1000, 2463]
    assert ss.mixed([3], 7) == [3, 3, 1]


def _qdesc(calls, interval, offset, tmin, tmax, group, n_series):
    ca = (L.Call * len(calls))(*[(L.AGG_COUNT if f == "count" else {"sum": L.AGG_SUM, "min": L.AGG_MIN, "max": L.AGG_MAX,
                                   "first": L.AGG_FIRST, "last": L.AGG_LAST}[f], c) for f, c in calls])
    gm = L.GROUP_ALL if group == "all" else L.GROUP_PER_SERIES
    d = L.QueryDesc(interval, offset, tmin, tmax, 1, len(calls), ca, 0, None, gm, n_series if gm == L.GROUP_PER_SERIES else 0, None, 0,
                    L.Q_STRICT_ORDER)
    d._keep = ca
    return d


CUTS = {"1000": lambda n: ss.mixed([1000], n), "1024": lambda n: ss.mixed([1024], n), "3": lambda n: ss.mixed([3], n),
        "1_2_33": lambda n: ss.mixed([1, 2, 33], n), "4096_1": lambda n: ss.mixed([4096, 1], n), "whole": lambda n: [n]}


@pytest.mark.parametrize("cut", list(CUTS))
def test_window_model_agrees_with_the_oracle(cut):
    """three series of 5000 rows (const-delta and irregular times, nulls in some columns), ties of values inside windows (f_lo,
    ints, bools) and of times across series (the same 1 s grid): every call the model answers, per series and for one tagset"""
    rng = np.random.default_rng(11)
    kinds = ["f_hi", "f_lo", "i_s8b", "bool", "i_wide"]
    types = ss.types_of(kinds)
    n = 5000
    series = [ss.series_rows(rng, n, kinds, [0, 0.2, 0.1, 0, 0]), ss.series_rows(rng, n, kinds, [0.05, 0, 0, 0.3, 0]),
              ss.series_rows(rng, n, kinds, 0.0, t0=ss.T0 + 333 * SEC + 17, irregular=True)]
    d = ss.shard_desc(series, types, [CUTS[cut](n) for _ in series])
    tmax_all = max(int(s["times"][-1]) for s in series)
    for iv, off, tmin, tmax in ((60 * SEC, 0, ss.T0, tmax_all), (7 * SEC, 3 * SEC, ss.T0 + 1234 * SEC + 5, ss.T0 + 3456 * SEC),
                                (3600 * SEC, -13 * SEC, ss.T0, tmax_all), (0, 0, ss.T0 + 10 * SEC, ss.T0 + 4321 * SEC)):
        for group in ("all", "series"):
            groups = [0, 0, 0] if group == "all" else [0, 1, 2]
            for col, typ in enumerate(types):
                funcs = ["count", "min", "max", "first", "last"] + ([] if typ == L.TYPE_BOOL else ["sum"])
                for calls in ([(f, col)] for f in funcs):
                    ref = oracle.scan(d, _qdesc(calls, iv, off, tmin, tmax, group, 3), threads=1)
                    model = ss.window_model(series, col, typ, iv, off, tmin, tmax, groups)
                    ss.check_against_model(ref, calls, model, typ, f"{cut} iv={iv} {group} {calls}")
                multi = [(f, col) for f in funcs]
                ref = oracle.scan(d, _qdesc(multi, iv, off, tmin, tmax, group, 3), threads=1)
                ss.check_against_model(ref, multi, ss.window_model(series, col, typ, iv, off, tmin, tmax, groups), typ,
                                       f"{cut} iv={iv} {group} multi c{col}")
