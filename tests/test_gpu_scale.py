"""Parity at the sizes BASELINE.json names (not only at toy sizes):

* configs[0]: 100 series x 10k float64 points, mean (sum, count) GROUP BY time(1m) — the reference's CPU-runnable case.
* a 1/50 slice of configs[1]: 100 of its 5000 series x 10^6 points, G-hi and G-lo, sum/count/max GROUP BY time(1m), against the oracle on
  the identical synthetic shard (same seed): strict order bitwise, folded order 1e-12 on float sums and bitwise on the rest,
  per-series grouping bitwise.
"""
import os

import numpy as np
import pytest

import oracle
from opengemini_b200 import AggQuery, Shard
from opengemini_b200 import _lib as L

pytestmark = pytest.mark.gpu
T0, SEC = 1_700_000_000_000_000_000, 1_000_000_000


@pytest.fixture(scope="module", autouse=True)
def _device():
    Shard.init(0)


def _cmp(got, ref, calls, exact_sum, label):
    for k, (f, _c) in enumerate(calls):
        rv = ref["cols"][k]["valid"].astype(bool)
        assert np.array_equal(got["cols"][k]["valid"].astype(bool), rv), (label, f)
        g, r = got["cols"][k]["values"].view(np.uint64)[rv], ref["cols"][k]["values"][rv]
        if f == "sum" and not exact_sum:
            assert np.allclose(g.view(np.float64), r.view(np.float64), rtol=1e-12, atol=0), (label, f)
        else:
            assert np.array_equal(g, r), (label, f)


def test_config0_100_series_x_10k_points_mean_group_by_1m():
    cols = [(L.TYPE_FLOAT, L.SYNTH_F_HI, 0)]
    sh = Shard.synth(100, 10_000, cols, t0=T0, dt=SEC, seed=2024)
    hs = oracle.HostShard(100, 10_000, cols, t0=T0, dt=SEC, seed=2024)
    calls = [("sum", 0), ("count", 0)]
    tmax = T0 + 9_999 * SEC
    for flags, exact in ((L.Q_STRICT_ORDER, True), (0, False), (L.Q_NO_FAST | L.Q_STRICT_ORDER, True), (L.Q_NO_FUSED, True)):
        q = AggQuery(sh, calls, 60 * SEC, T0, tmax, flags=flags).run()
        ref = oracle.scan(hs.desc, q.desc, threads=1)
        _cmp(q.dense_host(), ref, calls, exact, f"config0 flags={flags}")
        if flags == 0:  # the mean the user sees
            d = q.dense_host()
            mean = d["cols"][0]["values"] / d["cols"][1]["values"]
            rmean = ref["cols"][0]["values"].view(np.float64) / ref["cols"][1]["values"].view(np.int64)
            assert np.allclose(mean, rmean, rtol=1e-12, atol=0) and d["n_buckets"] == 167
        q.close()
    sh.close()


@pytest.mark.parametrize("dist", ["hi", "lo"])
def test_slice_of_config1_100_series_x_1M_points(dist):
    n_series, rows = 100, 1_000_000
    cols = [(L.TYPE_FLOAT, L.SYNTH_F_HI if dist == "hi" else L.SYNTH_F_LO, 0)]
    sh = Shard.synth(n_series, rows, cols, t0=T0, dt=SEC, seed=77)
    threads = max(1, min(16, len(os.sched_getaffinity(0))))
    hs = oracle.HostShard(n_series, rows, cols, t0=T0, dt=SEC, seed=77, threads=threads)
    assert sh.info()["page_bytes"] == sum(int(np.ctypeslib.as_array(hs.desc.columns[0].page_len, shape=(hs.desc.n_segments,)).sum()) for _ in [0]) + \
        int(np.ctypeslib.as_array(hs.desc.time_page_len, shape=(hs.desc.n_segments,)).sum())
    calls = [("sum", 0), ("count", 0), ("max", 0)]
    tmax = T0 + (rows - 1) * SEC
    q = AggQuery(sh, calls, 60 * SEC, T0, tmax, flags=L.Q_STRICT_ORDER).run()
    ref = oracle.scan(hs.desc, q.desc, threads=1)  # one cursor: the reference's fold order
    assert q.dense_host()["n_buckets"] == 16667
    _cmp(q.dense_host(), ref, calls, True, f"{dist} strict")
    q.close()
    q = AggQuery(sh, calls, 60 * SEC, T0, tmax).run()
    assert q.stats()["path"] == 3 and q.stats()["per_series_cells_used"] == 0
    _cmp(q.dense_host(), ref, calls, False, f"{dist} folded")
    q.close()
    # per-series grouping: every series is one cursor in the oracle too -> any thread count gives the same bits
    q = AggQuery(sh, calls, 60 * SEC, T0, tmax, group="series").run()
    refs = oracle.scan(hs.desc, q.desc, threads=threads)
    _cmp(q.dense_host(), refs, calls, True, f"{dist} per series")
    q.close()
    sh.close()
