"""What short segments cost the query path, and what compacting them back into full segments (og_shard_compact) costs.

    python tools/bench_compact.py [--series 2000] [--rows 1000000] [--flushes 50] [--flush-rows 20] [--query-reps 5]

The base shard is device-synthesised (og_shard_synth, float64 G-hi, 1 s cadence, 1000-row segments), as in tools/bench_append.py.
`flushes` ordered files of `flush-rows` rows per series follow, each appended with og_shard_append_files: every flush adds a
short segment to every series.  Measured: SELECT sum, count, max GROUP BY time(1m) over the whole shard before compaction (first
and steady runs, path), og_shard_compact (host wall clock around the synchronised call, compact_ms, og_compact_info), the first
query after it (which includes the interleaved-copy rebuild) and steady queries; the kernels of the pass (torch.profiler:
k_append_gather against a device-to-device copy of the same bytes); the same at flush-rows = 1000, where there is nothing to
do.  The answers before and after are checked: count, max and validity bitwise, sums to 1e-12 relative.  Prints one JSON line
with the card, its power limit and SM clock.  Needs a GPU; writes nothing.
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


def timed(fn):
    t = time.perf_counter()
    r = fn()
    return r, (time.perf_counter() - t) * 1e3


def desc_of(ex):
    nc = ex["col_types"].size
    return Shard.desc(ex["data"], ex["sids"], ex["series_seg_begin"], ex["seg_tmin"], ex["seg_tmax"],
                      [(f"f{c}", int(ex["col_types"][c]), ex["page_off"][c], ex["page_len"][c]) for c in range(nc)],
                      ex["page_off"][nc], ex["page_len"][nc])


def queries(sh, tmax, reps):
    """first run (plan + interleaved-copy build) and steady runs of the query; the answer of the last run"""
    q = AggQuery(sh, CALLS, 60 * SEC, T0, tmax)
    _r, first = timed(q.run)
    steady = [timed(q.run)[1] for _ in range(reps)]
    st = q.stats()
    d = q.dense_host()
    ans = [(c["valid"].copy(), c["values"].view(np.uint64).copy()) for c in d["cols"]]
    q.close()
    return dict(first_ms=first, steady_ms_min=min(steady), steady_ms=steady, path=st["path"], rows=st["rows_decoded"]), ans


def same_answers(a, b):
    for k, ((va, xa), (vb, xb)) in enumerate(zip(a, b)):
        assert np.array_equal(va, vb), ("validity", CALLS[k])
        if CALLS[k][0] == "sum":
            fa, fb = xa[va.astype(bool)].view(np.float64), xb[vb.astype(bool)].view(np.float64)
            assert np.all(np.abs(fa - fb) <= 1e-12 * np.maximum(1.0, np.abs(fb))), "sums differ beyond 1e-12"
        else:
            assert np.array_equal(xa, xb), CALLS[k]


def kernel_us(prof):
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


def scenario(a, flush_rows, profile_pass):
    sh = Shard.synth(a.series, a.rows, COLS, t0=T0, dt=SEC, seed=1001)
    for i in range(a.flushes):
        src = Shard.synth(a.series, flush_rows, COLS, t0=T0 + (a.rows + i * flush_rows) * SEC, dt=SEC, seed=2000 + i)
        d = desc_of(src.export())
        src.close()
        sh.append_files([(d, False)])
    L.lib().og_release_cached_memory()
    tmax = T0 + (a.rows + a.flushes * flush_rows) * SEC
    out = dict(flush_rows=flush_rows, flushes=a.flushes, info_before=sh.info())
    out["query_before"], before = queries(sh, tmax, a.query_reps)
    prof = None
    if profile_pass:
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            ci, wall = timed(sh.compact)
    else:
        ci, wall = timed(sh.compact)
    out["compact"] = dict(wall_ms=wall, **ci)
    out["info_after"] = sh.info()
    out["query_after"], after = queries(sh, tmax, a.query_reps)
    same_answers(after, before)
    for k in ("n_rows", "tmin", "tmax"):
        assert out["info_after"][k] == out["info_before"][k], k
    if prof is not None:
        ku = kernel_us(prof)
        pages = out["info_after"]["page_bytes"]
        gather_ms = sum(v for k, v in ku.items() if "k_append_gather" in k) / 1e3
        copy = d2d_ms(pages)
        out["kernels_ms"] = {k: v / 1e3 for k, v in sorted(ku.items(), key=lambda kv: -kv[1])[:10]}
        out["gather"] = dict(live_page_bytes=pages, k_append_gather_ms=gather_ms, d2d_copy_ms=copy,
                             gather_GBps=2 * pages / (gather_ms / 1e3) / 1e9 if gather_ms else None, d2d_GBps=2 * pages / (copy / 1e3) / 1e9)
    sh.close()
    L.lib().og_release_cached_memory()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--series", type=int, default=2000)
    ap.add_argument("--rows", type=int, default=1_000_000)
    ap.add_argument("--flushes", type=int, default=50)
    ap.add_argument("--flush-rows", type=int, default=20)
    ap.add_argument("--query-reps", type=int, default=5)
    a = ap.parse_args()
    Shard.init(0)
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    res = dict(card=card, base=f"{a.series} series x {a.rows} float64 rows (G-hi), 1 s cadence, 1000-row segments",
               query="SELECT sum, count, max GROUP BY time(1m), whole shard")
    res["short_flushes"] = scenario(a, a.flush_rows, True)
    res["full_flushes"] = scenario(a, 1000, False)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
