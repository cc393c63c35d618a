"""Cost of opening a shard from its file set (og_shard_open_files) on a configs[1]-shaped shard, and what the merge does to queries.

    python tools/bench_out_of_order.py [--series 5000] [--rows 200000] [--touch-every 100] [--late-rows 3000] [--reps 3]

The ordered file is a device-synthesised shard (og_shard_synth, float64 G-hi, 1 s cadence, 1000-row segments) exported to the host.
Two out-of-order files touch every `touch-every`-th series: one inserts rows between the ordered ones (half-second offsets), one
rewrites rows at the ordered times.  Prints one JSON line: the card and its power limit, og_shard_open against og_shard_open_files
on the ordered file alone, merge_ms and rewritten rows per second of the merge, and the query rate and og_stats.path of
SELECT sum, count, max GROUP BY time(1m) before and after the merge.  Needs a GPU; writes nothing.
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


def desc_of(ex, sids=None):
    nc = ex["col_types"].size
    return Shard.desc(ex["data"], ex["sids"] if sids is None else sids, ex["series_seg_begin"], ex["seg_tmin"], ex["seg_tmax"],
                      [(f"f{c}", int(ex["col_types"][c]), ex["page_off"][c], ex["page_len"][c]) for c in range(nc)],
                      ex["page_off"][nc], ex["page_len"][nc])


def timed(fn):
    t = time.perf_counter()
    r = fn()
    return r, (time.perf_counter() - t) * 1e3


def query_rate(sh, rows, tmax, reps):
    calls = [("sum", 0), ("count", 0), ("max", 0)]
    q = AggQuery(sh, calls, 60 * SEC, T0, tmax)
    q.run()  # plan + first-use builds
    ms = []
    for _ in range(reps):
        _r, m = timed(q.run)
        ms.append(m)
    st = q.stats()
    q.close()
    best = min(ms)
    return dict(ms_min=best, ms_all=ms, rows_per_s=rows / (best / 1e3), path=st["path"], per_series_cells_used=st["per_series_cells_used"])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--series", type=int, default=5000)
    ap.add_argument("--rows", type=int, default=200000)
    ap.add_argument("--touch-every", type=int, default=100)
    ap.add_argument("--late-rows", type=int, default=3000)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--query-reps", type=int, default=10)
    a = ap.parse_args()
    Shard.init(0)
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    cols = [(L.TYPE_FLOAT, L.SYNTH_F_HI, 0)]
    base = Shard.synth(a.series, a.rows, cols, t0=T0, dt=SEC, seed=1001)
    ordered = desc_of(base.export())
    n_rows = base.info()["n_rows"]
    tmax = T0 + (a.rows - 1) * SEC
    before = query_rate(base, n_rows, tmax, a.query_reps)
    base.close()
    # out-of-order files: series base+1 .. of the synthetic population, re-labelled with the touched series' sids
    touched = np.arange(0, a.series, a.touch_every, dtype=np.uint64) + 1
    mid = T0 + (a.rows // 2) * SEC
    ins = Shard.synth(touched.size, a.late_rows, cols, t0=mid + SEC // 2, dt=SEC, seed=2002)   # between the ordered rows
    rep = Shard.synth(touched.size, a.late_rows, cols, t0=mid + 500 * SEC, dt=SEC, seed=3003)  # at the ordered rows' times
    ooo1, ooo2 = desc_of(ins.export(), touched), desc_of(rep.export(), touched)
    ooo_segs = ins.info()["n_segments"] + rep.info()["n_segments"]
    ins.close(); rep.close()
    res = dict(card=card, shard=f"{a.series} series x {a.rows} float64 rows (G-hi), 1 s cadence, 1000-row segments",
               late=f"every {a.touch_every}th series ({touched.size}): {a.late_rows} inserted + {a.late_rows} rewritten rows each")
    opens, files1 = [], []
    for _ in range(a.reps):  # alternate the two open paths
        sh, m = timed(lambda: Shard.open_desc(ordered)); sh.close(); opens.append(m)
        sh, m = timed(lambda: Shard.open_files([(ordered, False)])); sh.close(); files1.append(m)
        L.lib().og_release_cached_memory()
    res["open_ms"] = dict(og_shard_open=opens, og_shard_open_files_one_file=files1)
    merges = []
    for _ in range(a.reps):
        sh, m = timed(lambda: Shard.open_files([(ordered, False), (ooo1, True), (ooo2, True)]))
        mi = sh.merge_info()
        span_rows = mi["out_of_order_rows"] + 1000 * (mi["segments_rewritten_in"] - ooo_segs)
        merges.append(dict(open_ms=m, merge_ms=mi["merge_ms"], rewritten_rows_in=span_rows, rewritten_rows_per_s=span_rows / (mi["merge_ms"] / 1e3), info=mi))
        if len(merges) < a.reps:
            sh.close()
            L.lib().og_release_cached_memory()
    res["merge"] = merges
    res["query_before"] = before
    res["query_after"] = query_rate(sh, sh.info()["n_rows"], tmax, a.query_reps)
    sh.close()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
