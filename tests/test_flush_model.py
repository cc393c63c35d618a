"""tests/flush_model.py, the CPU statement of the flush og_shard_append_rows runs, pinned by the reference's own cases (restated:
lib/record/column_sort_test.go TestColumnSortHelper_Sort / _SortSameTime with their int, float and bool columns, the string column
left out; engine/mutable/table_test.go:107-142 TestSplitRecordByTime) and by hand-worked ones.  No GPU needed."""
import numpy as np
import pytest

import flush_model as fm
from opengemini_b200 import _lib as L

INT, FLOAT, BOOL = L.TYPE_INT, L.TYPE_FLOAT, L.TYPE_BOOL


def _rec(times, vi, vb, vf, nil, nil_col):
    """the reference's buildRecord: columns vs (left out), vi, vb, vf; rows with nil[k] are null in column nil_col (0 = vs)"""
    n = len(times)
    ok = [np.ones(n, bool) for _ in range(4)]
    ok[nil_col] = ~np.asarray(nil, bool)
    return np.asarray(times, np.int64), {"vi": (INT, np.asarray(vi, np.int64), ok[1]),
                                         "vb": (BOOL, np.asarray(vb, np.uint8), ok[2]),
                                         "vf": (FLOAT, np.asarray(vf, np.float64), ok[3])}


def _values(cols, name):
    _t, v, ok = cols[name]
    return v[ok].tolist()


# ---------------------------------------------------------------- TestColumnSortHelper_Sort
@pytest.mark.parametrize("times,vi,vb,vf,exp_vi,exp_vb,exp_vf", [
    ([3, 1, 2, 5, 4], [3, 1, 2, 5, 4], [1, 1, 0, 0, 0], [.3, .1, .2, .5, .4], [1, 2, 3, 4, 5], [1, 0, 1, 0, 0], [.1, .2, .3, .4, .5]),
    ([5, 4, 3, 2, 1], [5, 4, 3, 2, 1], [0, 0, 0, 1, 1], [.5, .4, .3, .2, .1], [1, 2, 3, 4, 5], [1, 1, 0, 0, 0], [.1, .2, .3, .4, .5]),
    ([1, 2, 3, 4, 5], [1, 2, 3, 4, 5], [1, 1, 0, 0, 0], [.1, .2, .3, .4, .5], [1, 2, 3, 4, 5], [1, 1, 0, 0, 0], [.1, .2, .3, .4, .5]),
])
def test_column_sort_helper_sort(times, vi, vb, vf, exp_vi, exp_vb, exp_vf):
    t, cols = fm.sort_dedup(*_rec(times, vi, vb, vf, [False] * 5, 0))
    assert t.tolist() == [1, 2, 3, 4, 5]
    assert _values(cols, "vi") == exp_vi and _values(cols, "vb") == exp_vb and _values(cols, "vf") == exp_vf


@pytest.mark.parametrize("nil_col", [0, 1, 2, 3])
def test_column_sort_helper_sort_with_nulls(nil_col):
    t, cols = fm.sort_dedup(*_rec([1, 2, 5, 3, 4], [1, 2, 5, 3, 4], [1, 1, 0, 0, 0], [.1, .2, .5, .3, .4], [False, True, False, True, False], nil_col))
    assert t.tolist() == [1, 2, 3, 4, 5]
    exp = {"vi": [1, 2, 3, 4, 5], "vb": [1, 1, 0, 0, 0], "vf": [.1, .2, .3, .4, .5]}
    if nil_col == 1:
        exp["vi"] = [1, 4, 5]
    if nil_col == 2:
        exp["vb"] = [1, 0, 0]
    if nil_col == 3:
        exp["vf"] = [.1, .4, .5]
    for name, want in exp.items():
        assert _values(cols, name) == want, name


# ---------------------------------------------------------------- TestColumnSortHelper_SortSameTime
@pytest.mark.parametrize("nil_col,exp_vi", [(1, [1, 2, 3, 4, 55]), (0, [1, 22, 3, 4, 55])])
def test_column_sort_helper_sort_same_time(nil_col, exp_vi):
    t, cols = fm.sort_dedup(*_rec([3, 1, 2, 5, 4, 2, 5], [3, 1, 2, 5, 4, 22, 55], [1, 1, 0, 0, 0, 1, 0], [.3, .1, .2, .5, .4, .22, .55],
                                  [False, False, False, True, False, True, False], nil_col))
    assert t.tolist() == [1, 2, 3, 4, 5]
    assert _values(cols, "vi") == exp_vi
    assert _values(cols, "vb") == [1, 1, 1, 0, 0]
    assert _values(cols, "vf") == [.1, .22, .3, .4, .55]


# ---------------------------------------------------------------- TestSplitRecordByTime
def test_split_record_by_time():
    t = np.arange(1, 6, dtype=np.int64)
    cols = {"a1": (INT, np.arange(1, 6), np.ones(5, bool)), "a2": (FLOAT, np.array([1.1, 2.1, 3.1, 4.1, 5.1]), np.ones(5, bool))}
    order, unorder = fm.split(t, cols, 3)
    assert order[0].tolist() == [4, 5] and unorder[0].tolist() == [1, 2, 3]
    assert _values(order[1], "a1") == [4, 5] and _values(unorder[1], "a1") == [1, 2, 3]


def test_split_record_by_time_drops_an_all_null_column():
    t = np.array([1, 2, 3, 7, 8], np.int64)
    cols = {"a1": (INT, np.array([0, 0, 0, 4, 5]), np.array([0, 0, 0, 1, 1], bool)),
            "a2": (FLOAT, np.array([1.1, 2.1, 3.1, 0, 0]), np.array([1, 1, 1, 0, 0], bool))}
    order, unorder = fm.split(t, cols, 4)
    assert order[0].size == 2 and unorder[0].size == 3
    assert sorted(order[1]) == ["a1"] and sorted(unorder[1]) == ["a2"]  # Len() == 2: one field and the time column


@pytest.mark.parametrize("last, side", [(0, 0), (8, 1)])
def test_split_drops_an_all_null_column_when_every_row_is_on_one_side(last, side):
    """the flush's documented deviation: ts_table.go:243-248 returns the record itself when every row falls on one side, so the
    reference keeps a column null in every row; the flush drops it there too, as it does when the rows straddle the last time"""
    t = np.array([1, 2, 3, 7, 8], np.int64)
    cols = {"a1": (INT, np.arange(5), np.ones(5, bool)), "a2": (FLOAT, np.zeros(5), np.zeros(5, bool))}
    parts = fm.split(t, cols, last)
    assert parts[1 - side] is None
    assert parts[side][0].tolist() == t.tolist() and sorted(parts[side][1]) == ["a1"]


# ---------------------------------------------------------------- hand-worked
def test_a_null_never_replaces_a_value_and_the_last_value_wins():
    t = np.array([10, 10, 10, 20, 10], np.int64)
    v = np.array([1, 2, 3, 4, 5], np.int64)
    ok = np.array([1, 1, 0, 1, 0], bool)           # time 10: 1, 2, null, null in arrival order -> 2
    b_ok = np.array([0, 0, 0, 1, 0], bool)          # time 10 never has a value -> null
    ts, cols = fm.sort_dedup(t, {"v": (INT, v, ok), "b": (BOOL, np.ones(5, np.uint8), b_ok)})
    assert ts.tolist() == [10, 20]
    assert cols["v"][1].tolist() == [2, 4] and cols["v"][2].tolist() == [True, True]
    assert cols["b"][2].tolist() == [False, True]


def test_flush_splits_at_each_series_last_time_and_counts_replaced_rows():
    batch = {7: dict(times=np.array([5, 1, 9, 5, 3], np.int64), cols={"v": (FLOAT, np.arange(5.0), np.ones(5, bool))}),
             3: dict(times=np.array([2, 2], np.int64), cols={"v": (FLOAT, np.array([1.0, 2.0]), np.array([1, 0], bool))})}
    ordered, ooo, replaced = fm.flush(batch, {7: 5})
    assert replaced == 2
    assert ordered[7]["times"].tolist() == [9] and ooo[7]["times"].tolist() == [1, 3, 5]
    assert ooo[7]["cols"]["v"][1].tolist() == [1.0, 4.0, 3.0]   # time 5: arrival rows 0 and 3, the later wins
    assert ordered[3]["times"].tolist() == [2] and 3 not in ooo   # a sid the shard lacks: every row ordered
    assert [ooo_ for _f, ooo_ in fm.files(batch, {7: 5})] == [False, True]
    assert [ooo_ for _f, ooo_ in fm.files(batch, {7: 100, 3: 100})] == [True]


@pytest.mark.parametrize("n,segs", [(1, [1]), (999, [999]), (1000, [1000]), (1001, [1000, 1]), (2500, [1000, 1000, 500])])
def test_each_part_is_cut_into_1000_row_segments_from_its_first_row(n, segs):
    t = np.arange(n, dtype=np.int64) * 10
    ok = np.ones(n, bool)
    ok[::2] = False
    names, _types, series = fm.file_pages({1: dict(times=t, cols={"v": (INT, np.arange(n), ok)})})
    (_sid, ss), = series
    assert [int((hi - lo) // 10 + 1) for lo, hi, _p, _t in ss] == segs
    assert all("v" in p for _lo, _hi, p, _t in ss)  # a kept column has a page in every segment, an all-null one included
