"""The restated file-set read (tests/oracle_files.py): the reference's record-merge KATs, and agreement with a plain-Python model
of the row rule on seeded random file sets (no GPU)."""
import numpy as np
import pytest

import oracle_files as F
from opengemini_b200 import _lib as L

TYPE_STRING = 4
SCHEMA = [("boolean", L.TYPE_BOOL), ("float", L.TYPE_FLOAT), ("int", L.TYPE_INT), ("string", TYPE_STRING)]


def gen_row_rec(schema, iv, ib, fv, fb, sv, sb, bv, bb, times):
    """genRowRec (lib/record/record_test.go:28-80): per column a 0/1 bitmap and the values."""
    r = F.rec_new(schema)
    src = {"int": (iv, ib), "float": (fv, fb), "string": (sv, sb), "boolean": (bv, bb)}
    for name, _t in schema:
        vals, bm = src[name]
        r["cols"][name] = [vals[i] if bm[i] else None for i in range(len(times))]
    r["times"] = list(times)
    return r


def same(a, b):
    return a["times"] == b["times"] and all(a["cols"].get(n) == b["cols"].get(n) for n, _t in b["schema"]) and \
        sorted(n for n, _ in a["schema"]) == sorted(n for n, _ in b["schema"])


def test_kat_different_schema_one_row_case1():  # record_test.go:319-360
    old = gen_row_rec([("boolean", L.TYPE_BOOL), ("int", L.TYPE_INT)], [200], [1], [], [0], [], [0], [False], [1], [1])
    new = gen_row_rec([("float", L.TYPE_FLOAT), ("int", L.TYPE_INT), ("string", TYPE_STRING)], [100], [1], [1.3], [1], ["test"], [1], [], [0], [1])
    exp = gen_row_rec(SCHEMA, [100], [1], [1.3], [1], ["test"], [1], [False], [1], [1])
    m = F.rec_new()
    F.merge_record(m, new, old)
    assert same(m, exp)


def test_kat_same_schema_multi_rows_case3():  # record_test.go:729-762
    old = gen_row_rec(SCHEMA, [200, 300, 0, 400, 500, 600, 700], [1, 1, 0, 1, 1, 1, 1], [2.3, 0, 3.3, 0, 4.3, 5.3, 0], [1, 0, 1, 0, 1, 1, 0],
                      ["", "hello", "", "", "world", "", "test"], [0, 1, 0, 0, 1, 0, 1], [False, False, True, False, True, False, False],
                      [0, 0, 1, 0, 1, 1, 0], [31, 32, 33, 34, 45, 46, 47])
    new = gen_row_rec(SCHEMA, [1000, 0, 1100, 1200, 1300, 1400, 0], [1, 0, 1, 1, 1, 1, 0], [1001.3, 1002.4, 0, 1003.5, 0, 0, 2000.6],
                      [1, 1, 0, 1, 0, 0, 1], ["", "helloNew", "worldNew", "testNew1", "", "testNew2", "testNew3"], [0, 1, 1, 1, 0, 1, 1],
                      [True, True, False, True, False, False, True], [1, 1, 1, 1, 0, 1, 1], [31, 32, 33, 34, 45, 46, 47])
    exp = gen_row_rec(SCHEMA, [1000, 300, 1100, 1200, 1300, 1400, 700], [1] * 7, [1001.3, 1002.4, 3.3, 1003.5, 4.3, 5.3, 2000.6], [1] * 7,
                      ["", "helloNew", "worldNew", "testNew1", "world", "testNew2", "testNew3"], [0, 1, 1, 1, 1, 1, 1],
                      [True, True, False, True, True, False, True], [1] * 7, [31, 32, 33, 34, 45, 46, 47])
    m = F.rec_new()
    F.merge_record(m, new, old)
    assert same(m, exp)


def _one(i, f, s, b, t):
    return gen_row_rec(SCHEMA, [i], [1], [f], [1], [s], [1], [b], [1], [t])


def test_kat_limit_rows_case1():  # record_test.go:1756-1779: equal times, limit 1 -> the older row, positions (0, 1)
    old, new = _one(200, 2.3, "hello", False, 1), _one(100, 1.3, "world", True, 2)
    m = F.rec_new()
    assert F.merge_record_limit_rows(m, new, old, 0, 0, 1) == (0, 1)
    assert same(m, old)


def test_kat_limit_rows_case2():  # record_test.go:1806-1829
    old, new = _one(200, 2.3, "hello", False, 3), _one(100, 1.3, "world", True, 2)
    m = F.rec_new()
    assert F.merge_record_limit_rows(m, new, old, 0, 0, 1) == (1, 0)
    assert same(m, new)


def test_kat_by_max_time_of_old_rec_case1():  # record_test.go:2162-2188
    old = gen_row_rec(SCHEMA, [200, 300, 0, 400, 500, 600, 700], [1, 1, 0, 1, 1, 1, 1], [2.3, 0, 3.3, 0, 4.3, 5.3, 0], [1, 0, 1, 0, 1, 1, 0],
                      ["", "hello", "", "", "world", "", "test"], [0, 1, 0, 0, 1, 0, 1], [False, False, True, False, True, False, False],
                      [0, 0, 1, 0, 1, 1, 0], [31, 32, 33, 34, 45, 46, 47])
    new = gen_row_rec(SCHEMA, [1000, 0, 1100, 1200, 1300, 1400, 0], [1, 0, 1, 1, 1, 1, 0], [1001.3, 1002.4, 0, 1003.5, 0, 0, 2000.6],
                      [1, 1, 0, 1, 0, 0, 1], ["", "helloNew", "worldNew", "testNew1", "", "testNew2", "testNew3"], [0, 1, 1, 1, 0, 1, 1],
                      [True, True, False, True, False, False, True], [1, 1, 1, 1, 0, 1, 1], [48, 49, 50, 51, 52, 53, 54])
    exp = gen_row_rec(SCHEMA, [300, 0, 400, 500, 600, 700], [1, 0, 1, 1, 1, 1], [0, 3.3, 0, 4.3, 5.3, 0], [0, 1, 0, 1, 1, 0],
                      ["hello", "", "", "world", "", "test"], [1, 0, 0, 1, 0, 1], [False, True, False, True, False, False], [0, 1, 0, 1, 1, 0],
                      [32, 33, 34, 45, 46, 47])
    m = F.rec_new()
    assert F.merge_record_by_max_time_of_old_rec(m, new, old, 0, 1, 1000) == (0, 7)
    assert same(m, exp)


# ---------------------------------------------------------------- random file sets against a plain-Python model
def _model(files):
    order = sorted(range(len(files)), key=lambda i: (files[i][1], i))
    rows = {}
    for i in order:
        for sid, s in files[i][0].items():
            r = rows.setdefault(sid, {})
            for k, t in enumerate(s["times"].tolist()):
                row = r.setdefault(t, {})
                for n, (_ty, v, ok) in s["cols"].items():
                    if ok[k]:
                        row[n] = v[k].item()
    return rows


def _random(seed, layout):
    rng = np.random.default_rng(seed)
    T0 = 10_000

    def series(t, names, null_p):
        cols = {}
        for n in names:
            ty = {"f": L.TYPE_FLOAT, "i": L.TYPE_INT, "b": L.TYPE_BOOL}[n[0]]
            v = rng.normal(0, 10, t.size) if ty == L.TYPE_FLOAT else rng.integers(-50, 50, t.size) if ty == L.TYPE_INT else rng.integers(0, 2, t.size).astype(np.uint8)
            cols[n] = (ty, v, rng.random(t.size) >= null_p)
        return dict(times=np.asarray(t, np.int64), cols=cols)

    files = []
    for ooo in layout:
        f = {}
        for sid in range(1, 7):
            if rng.random() < 0.3:
                continue
            if ooo:
                t = np.unique(T0 + rng.integers(-100, 3200, int(rng.integers(5, 300))))
                names = [n for n in ("f1", "i1", "b1") if rng.random() < 0.7] or ["f1"]
            else:
                k = len(files)
                t = T0 + np.arange(k * 1100, k * 1100 + 1100) * 2  # ordered files in time order, never overlapping
                names = ["f1", "i1", "b1"]
            f[sid] = series(t, names, 0.25 if ooo else 0.05)
        files.append((f, ooo))
    return files


@pytest.mark.parametrize("seed,layout", [(1, (False, True)), (2, (False, True, True)), (3, (False, True, False, True)),
                                          (4, (True, False, True)), (5, (False, False, True, True, True))])
def test_file_set_read_equals_the_model(seed, layout):
    """Duplicates across ordered and out-of-order files and across out-of-order files, nulls in the newer rows, columns present
    in only some files, series only the out-of-order files hold, ordered files after out-of-order ones in file order."""
    files = _random(seed, layout)
    model = _model(files)
    recs = F.read_files(files, {"tmin": -(1 << 62), "tmax": 1 << 62})
    assert sorted(recs) == sorted(model)
    for sid, rs in recs.items():
        times = [t for r in rs for t in r["times"]]
        assert times == sorted(model[sid]), sid
        assert all(F.rows(r) <= F.CHUNK_SIZE_NUM for r in rs)
        for r in rs:
            for k, t in enumerate(r["times"]):
                got = {n: c[k] for n, c in r["cols"].items() if c[k] is not None}
                assert got == model[sid][t], (sid, t)
