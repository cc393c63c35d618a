"""SURVEY §8f row 3 / configs[4] shape at test size: decode -> per-series re-aggregation -> re-encode -> read back.

og_downsample's pages (through downsample(), the pass bench.py times) are checked three ways: (1) decoded with the ORACLE they
hold exactly the oracle's per-series aggregates, (2) byte for byte they are what the oracle's encoders write for those values,
(3) reopened as a shard on the GPU, coarser queries over them agree with the same queries over the source shard.
"""
import numpy as np
import pytest

import oracle
from opengemini_b200 import _lib as L

T0, SEC = 1_700_000_000_000_000_000, 1_000_000_000
pytestmark = pytest.mark.gpu


def test_downsample_reencode_roundtrip():
    _roundtrip(L.TYPE_FLOAT, L.SYNTH_F_HI, 0)


@pytest.mark.parametrize("typ,dist,nulls", [(L.TYPE_INT, L.SYNTH_INT_WALK, 0), (L.TYPE_FLOAT, L.SYNTH_F_HI, 400)], ids=["int", "float_nulls"])
def test_downsample_reencode_roundtrip_int_and_nulls(typ, dist, nulls):
    _roundtrip(typ, dist, nulls)


def _roundtrip(typ, dist, nulls):
    """Column 1 of a shard whose column 0 is bool.  With nulls, 2-second windows include windows whose rows are all null: the
    row rule drops them (count is not valid there, and neither is any other call), and every kept window has all six cells
    valid, so every page is a page without nulls."""
    from opengemini_b200 import AggQuery, Shard
    from opengemini_b200.downsample import OUT_CALLS, downsample

    ns, rows, ivl = 6, 5000, 2 * SEC  # 2500 windows per series -> 3 output segments per series (1000-row limit)
    cols = [(L.TYPE_BOOL, L.SYNTH_BOOL, 0), (typ, dist, nulls)]
    sh = Shard.synth(ns, rows, cols, t0=T0, dt=SEC, seed=9)
    hs = oracle.HostShard(ns, rows, cols, t0=T0, dt=SEC, seed=9)
    tmin, tmax = T0 + 3 * SEC, T0 + (rows - 7) * SEC
    out = downsample(sh, 1, ivl, tmin, tmax)
    assert [c[0] for c in out["columns"]] == [f"{f}_f1" for f in OUT_CALLS]
    assert [c[1] for c in out["columns"]] == [L.TYPE_INT if f == "count" else typ for f in OUT_CALLS]

    # expectation: the oracle's per-series aggregates
    funcs = [L.AGG_MIN, L.AGG_MAX, L.AGG_SUM, L.AGG_COUNT, L.AGG_FIRST, L.AGG_LAST]
    ca = (L.Call * 6)(*[(f, 1) for f in funcs])
    qd = L.QueryDesc(ivl, 0, tmin, tmax, 1, 6, ca, 0, None, L.GROUP_PER_SERIES, ns, None, 0, 0)
    ref = oracle.scan(hs.desc, qd, threads=1)
    nb = ref["n_buckets"]
    kept = ref["cols"][3]["valid"].astype(bool)
    for k, f in enumerate(OUT_CALLS):
        assert np.array_equal(ref["cols"][k]["valid"].astype(bool), kept), f
    # windows that hold rows (column 0 has no nulls) but no value of column 1
    n0 = (L.Call * 1)((L.AGG_COUNT, 0))
    has_rows = oracle.scan(hs.desc, L.QueryDesc(ivl, 0, tmin, tmax, 1, 1, n0, 0, None, L.GROUP_PER_SERIES, ns, None, 0, 0), threads=1)
    all_null = int((has_rows["cols"][0]["valid"].astype(bool) & ~kept).sum())
    assert (all_null > 0) == (nulls > 0), all_null
    data = out["data"].cpu().numpy()
    ssb = out["series_seg_begin"]
    assert ssb[-1] == len(out["seg_tmin"]) and out["rows"] == int(kept.sum())
    for s in range(ns):
        ok = kept[s * nb:(s + 1) * nb]
        want_t = (ref["start"] + np.arange(nb, dtype=np.int64) * ivl)[ok]
        got_t = []
        for g in range(ssb[s], ssb[s + 1]):
            tp = data[out["time_page_off"][g]:out["time_page_off"][g] + out["time_page_len"][g]]
            got_t.append(oracle.time_page_decode(tp))
            assert out["seg_tmin"][g] == got_t[-1][0] and out["seg_tmax"][g] == got_t[-1][-1]
        assert np.array_equal(np.concatenate(got_t), want_t), s
        for k, f in enumerate(OUT_CALLS):
            _name, ctyp, po, pl = out["columns"][k]
            want = ref["cols"][k]["values"][s * nb:(s + 1) * nb][ok]
            got, at = [], 0
            for g in range(ssb[s], ssb[s + 1]):
                page = data[po[g]:po[g] + pl[g]]
                v, valid = oracle.field_page_decode(ctyp, page)
                assert valid.all()
                got.append(v.view(np.uint64))
                # byte parity with the restated reference encoder on the same values
                cells = want[at:at + v.size].view(np.float64 if ctyp == L.TYPE_FLOAT else np.int64)
                assert np.array_equal(oracle.field_page_encode(ctyp, cells), page), (s, f, g)
                at += v.size
            assert np.array_equal(np.concatenate(got), want), (s, f)  # bit-exact, float sums included

    # reopen the downsampled shard and query it: 1-minute aggregates from the 2-second partials
    host = data[:out["data_len"]].copy()
    ds = Shard.open(host, out["sids"], ssb, out["seg_tmin"], out["seg_tmax"], out["columns"], out["time_page_off"], out["time_page_len"])
    # (downsampled rows carry their window start as time, so the comparison range is aligned to the 2-second windows)
    qmin, qmax = T0 + 4 * SEC, T0 + 4989 * SEC
    q1 = AggQuery(ds, [("min", 0), ("max", 1), ("sum", 2), ("sum", 3)], 60 * SEC, qmin, qmax).run().dense_host()
    q0 = AggQuery(sh, [("min", 1), ("max", 1), ("sum", 1), ("count", 1)], 60 * SEC, qmin, qmax).run().dense_host()
    assert q1["n_buckets"] == q0["n_buckets"]
    for k in range(4):
        assert np.array_equal(q1["cols"][k]["valid"], q0["cols"][k]["valid"])
    m = q0["cols"][0]["valid"].astype(bool)
    assert np.array_equal(q1["cols"][0]["values"][m], q0["cols"][0]["values"][m])  # min of mins
    assert np.array_equal(q1["cols"][1]["values"][m], q0["cols"][1]["values"][m])  # max of maxes
    assert np.array_equal(q1["cols"][3]["values"][m], q0["cols"][3]["values"][m])  # sum of counts == count
    a, b = q1["cols"][2]["values"][m], q0["cols"][2]["values"][m]
    assert np.all(np.abs(a - b) <= 1e-9 * np.abs(b))  # re-associated float sums: north_star tolerance

    # the handle behind downsample() opens in place (OG_SHARD_DEVICE_DATA) and answers whole-range queries like the source
    got = sh.downsample(1, ivl, tmin, tmax)
    assert got.export().tobytes() == data[:out["data_len"]].tobytes()
    x = got.open()
    q1 = AggQuery(x, [("sum", 3), ("min", 0), ("max", 1)], 0, tmin - ivl, tmax).run().dense_host()
    q0 = AggQuery(sh, [("count", 1), ("min", 1), ("max", 1)], 0, tmin, tmax).run().dense_host()
    for k in range(3):
        assert int(q1["cols"][k]["values"].view(np.uint64)[0]) == int(q0["cols"][k]["values"].view(np.uint64)[0]), k
    x.close(); got.close()
    # a range without rows: a shard with the source's series and no segments, not an error
    e = sh.downsample(1, ivl, T0 + 10_000 * SEC, T0 + 20_000 * SEC)
    assert e.rows == 0 and e.desc.n_segments == 0 and e.desc.n_series == ns and e.desc.n_columns == 6
    e.close()
    ds.close(); sh.close()
