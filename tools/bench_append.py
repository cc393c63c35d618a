"""Cost of appending flushed files to an open shard (og_shard_append_files) against reopening the whole file set.

    python tools/bench_append.py [--series 2000] [--rows 1000000] [--flush-rows 10000] [--touch-every 100] [--small-rows 200000]

The base shard is device-synthesised (og_shard_synth, float64 G-hi, 1 s cadence, 1000-row segments).  Flush 1 is an ordered file
of `flush-rows` rows per series after the base; flush 2 is the next ordered file plus an out-of-order file that inserts rows of
every `touch-every`-th series (half-second offsets) inside flush 1's range.  Every appended shard is checked against
og_shard_open_files over the whole set (og_shard_info; SELECT sum, count, max GROUP BY time(1m): bitwise after flush 1, count, max
and validity bitwise after flush 2, whose merged float sums may differ in rounding).  Prints one JSON line: the card and its power
limit, host wall clock around each synchronised append, the reopen it replaces, merge_info, the first query after each append
(timed before any other query touches the shard, so it includes the interleaved-copy rebuild) and steady queries, the kernels of the
first append (torch.profiler: k_append_gather alone against a device-to-device copy of the same bytes in the same run), and the
same append onto a base of `small-rows` rows per series.  Needs a GPU; writes nothing.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from opengemini_b200 import AggQuery, Shard  # noqa: E402
from opengemini_b200 import _lib as L  # noqa: E402

T0, SEC = 1_700_000_000_000_000_000, 1_000_000_000
COLS = [(L.TYPE_FLOAT, L.SYNTH_F_HI, 0)]
CALLS = [("sum", 0), ("count", 0), ("max", 0)]


def desc_of(ex, sids=None):
    nc = ex["col_types"].size
    return Shard.desc(ex["data"], ex["sids"] if sids is None else sids, ex["series_seg_begin"], ex["seg_tmin"], ex["seg_tmax"],
                      [(f"f{c}", int(ex["col_types"][c]), ex["page_off"][c], ex["page_len"][c]) for c in range(nc)],
                      ex["page_off"][nc], ex["page_len"][nc])


def timed(fn):
    t = time.perf_counter()
    r = fn()
    return r, (time.perf_counter() - t) * 1e3


def synth_desc(n_series, rows, t0, seed, dt=SEC, sids=None):
    sh = Shard.synth(n_series, rows, COLS, t0=t0, dt=dt, seed=seed)
    d = desc_of(sh.export(), sids)
    sh.close()
    return d


def dense(sh, tmax):
    q = AggQuery(sh, CALLS, 60 * SEC, T0, tmax).run()
    d = q.dense_host()
    q.close()
    return [(c["valid"].copy(), c["values"].view(np.uint64).copy()) for c in d["cols"]]


def query_times(sh, tmax, reps):
    q = AggQuery(sh, CALLS, 60 * SEC, T0, tmax)
    _r, first = timed(q.run)  # plan + interleaved-copy build
    steady = [timed(q.run)[1] for _ in range(reps)]
    st = q.stats()
    q.close()
    return dict(first_ms=first, steady_ms_min=min(steady), steady_ms=steady, path=st["path"], il_build_ms=st["il_build_ms"])


def kernel_us(prof):
    """device time per kernel name (microseconds) of a torch.profiler run"""
    out = {}
    for e in prof.key_averages():
        t = getattr(e, "device_time_total", None)
        if t is None:
            t = getattr(e, "cuda_time_total", 0)
        if t:
            out[e.key] = out.get(e.key, 0) + t
    return out


def d2d_ms(n_bytes):
    import torch
    a = torch.empty(n_bytes, dtype=torch.uint8, device="cuda")
    b = torch.empty_like(a)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ms = []
    for _ in range(3):
        e0.record(); b.copy_(a); e1.record(); e1.synchronize()
        ms.append(e0.elapsed_time(e1))
    del a, b
    torch.cuda.empty_cache()
    return min(ms)


def flushes(a, rows_before):
    t1 = T0 + rows_before * SEC
    f1 = synth_desc(a.series, a.flush_rows, t1, 11)
    f2 = synth_desc(a.series, a.flush_rows, t1 + a.flush_rows * SEC, 12)
    touched = np.arange(0, a.series, a.touch_every, dtype=np.uint64) + 1
    late = synth_desc(touched.size, a.flush_rows // 2, t1 + SEC // 2, 13, dt=2 * SEC, sids=touched)  # inserted and rewritten rows
    return f1, f2, late


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--series", type=int, default=2000)
    ap.add_argument("--rows", type=int, default=1_000_000)
    ap.add_argument("--flush-rows", type=int, default=10_000)
    ap.add_argument("--touch-every", type=int, default=100)
    ap.add_argument("--small-rows", type=int, default=200_000)
    ap.add_argument("--query-reps", type=int, default=5)
    a = ap.parse_args()
    Shard.init(0)
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    res = dict(card=card, base=f"{a.series} series x {a.rows} float64 rows (G-hi), 1 s cadence, 1000-row segments",
               flushes=f"{a.series} x {a.flush_rows} ordered rows; then the same plus an out-of-order file on every {a.touch_every}th series")
    f1, f2, late = flushes(a, a.rows)
    tmax = T0 + (a.rows + 2 * a.flush_rows) * SEC
    # ---- the reopen the append replaces (og_shard_open_files over the whole set), kept for the check ----
    base = Shard.synth(a.series, a.rows, COLS, t0=T0, dt=SEC, seed=1001)
    base_desc = desc_of(base.export())
    base.close()
    fresh, reopen1 = timed(lambda: Shard.open_files([(base_desc, False), (f1, False)]))
    want1, info1 = dense(fresh, tmax), fresh.info()
    fresh.close()
    fresh, reopen2 = timed(lambda: Shard.open_files([(base_desc, False), (f1, False), (f2, False), (late, True)]))
    want2, info2 = dense(fresh, tmax), fresh.info()
    fresh.close()
    del base_desc
    L.lib().og_release_cached_memory()
    res["reopen_ms"] = dict(after_flush1=reopen1, after_flush2=reopen2)
    # ---- the appends ----
    sh = Shard.synth(a.series, a.rows, COLS, t0=T0, dt=SEC, seed=1001)
    res["query_before"] = query_times(sh, tmax, a.query_reps)
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        _r, m1 = timed(lambda: sh.append_files([(f1, False)]))
    mi1 = sh.merge_info()
    after1 = query_times(sh, tmax, a.query_reps)  # the first query after the append, before the check below
    assert sh.info() == info1, (sh.info(), info1)
    got = dense(sh, tmax)
    assert all(np.array_equal(x[0], y[0]) and np.array_equal(x[1], y[1]) for x, y in zip(got, want1)), "flush 1: answers differ from the reopen"
    res["append_ordered"] = dict(wall_ms=m1, merge_ms=mi1["merge_ms"], after=after1)
    pages = sh.info()["page_bytes"]
    _r, m2 = timed(lambda: sh.append_files([(f2, False), (late, True)]))
    mi2 = sh.merge_info()
    after2 = query_times(sh, tmax, a.query_reps)
    got = dense(sh, tmax)
    i2 = sh.info()
    assert i2["n_rows"] == info2["n_rows"] and i2["tmin"] == info2["tmin"] and i2["tmax"] == info2["tmax"], (i2, info2)
    for k, (x, y) in enumerate(zip(got, want2)):  # sum, count, max: merged float sums may differ in rounding
        assert np.array_equal(x[0], y[0]), ("flush 2 validity", k)
        if CALLS[k][0] != "sum":
            assert np.array_equal(x[1], y[1]), ("flush 2", CALLS[k])
    res["append_with_out_of_order"] = dict(wall_ms=m2, merge_ms=mi2["merge_ms"], info=mi2, after=after2)
    sh.close()
    L.lib().og_release_cached_memory()
    # ---- the first append's kernels; k_append_gather against a device-to-device copy of the same live pages ----
    ku = kernel_us(prof)
    gather_ms = sum(v for k, v in ku.items() if "k_append_gather" in k) / 1e3
    copy = d2d_ms(pages)
    res["kernels_first_append_ms"] = {k: v / 1e3 for k, v in sorted(ku.items(), key=lambda kv: -kv[1])[:8]}
    res["gather"] = dict(live_page_bytes=pages, k_append_gather_ms=gather_ms, d2d_copy_ms=copy,
                         gather_GBps=2 * pages / (gather_ms / 1e3) / 1e9, d2d_GBps=2 * pages / (copy / 1e3) / 1e9,
                         kernels_ms=sum(ku.values()) / 1e3, merge_ms=mi1["merge_ms"])
    # ---- the same flush onto a smaller base: the host part does not follow the existing shard ----
    f1s, _f2s, _lates = flushes(a, a.small_rows)
    small = Shard.synth(a.series, a.small_rows, COLS, t0=T0, dt=SEC, seed=1001)
    _r, ms = timed(lambda: small.append_files([(f1s, False)]))
    res["append_ordered_small_base"] = dict(rows_per_series=a.small_rows, wall_ms=ms, merge_ms=small.merge_info()["merge_ms"])
    small.close()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
