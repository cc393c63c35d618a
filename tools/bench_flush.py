"""Cost of flushing memtable rows into an open shard on the device (og_shard_append_rows) against appending the same rows as
pre-encoded files (og_shard_append_files).

    python tools/bench_flush.py [--series 2000] [--rows 1000000] [--flush-rows 10000] [--query-reps 5]

The base shard is device-synthesised (og_shard_synth, float64 G-hi, 1 s cadence, 1000-row segments).  Two flushes of
`flush-rows` rows per series follow it:
  (a) the float column only, every row after the series' last time (ordered);
  (b) the float column plus a new integer and a new boolean column, 5 % nulls each, 1 % of the rows late (inside flush (a)'s
      range, half-second offsets) and 5 % repeating another row's time of the same series.
Rows are handed over in arrival order.  Prints one JSON line: the card and its power limit (read in this run), host wall clock
around each synchronised og_shard_append_rows with its phase_ms, the same two flushes as the files tests/flush_model.py writes for
them through og_shard_append_files on a twin base (the files are encoded beforehand by the oracle's C++ encoders called per
segment from Python, not by the Go encoders; that host time is reported as what it is and not timed into the append), the first
query after each flush and steady queries, and the kernels of flush (a) from torch.profiler in a separate run on a fresh base.
Answer check: og_shard_info and og_shard_merge_info of each flushed shard equal its twin's, and so does the SHA-256 of its whole
export (directory and data region: both appends gather the live pages in directory order).  Needs a GPU; writes nothing.
"""
import argparse
import hashlib
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import flush_model as fm  # noqa: E402
from bench_append import kernel_us, query_times, timed  # noqa: E402
from opengemini_b200 import Shard  # noqa: E402
from opengemini_b200 import _lib as L  # noqa: E402

T0, SEC = 1_700_000_000_000_000_000, 1_000_000_000
COLS = [(L.TYPE_FLOAT, L.SYNTH_F_HI, 0)]


def batch_a(rng, sids, rows, n):
    t = T0 + (rows + np.arange(n, dtype=np.int64)) * SEC
    ok = np.ones(n, bool)
    return {sid: dict(times=t, cols={"f0": (L.TYPE_FLOAT, rng.normal(100, 20, n), ok)}) for sid in sids}


def batch_b(rng, sids, rows, n):
    out = {}
    for sid in sids:
        t = T0 + (rows + n + np.arange(n, dtype=np.int64)) * SEC
        late = rng.random(n) < 0.01
        t[late] = T0 + (rows + rng.integers(0, n, int(late.sum()))) * SEC + SEC // 2
        dup = (rng.random(n) < 0.05) & ~late
        t[dup] = t[rng.integers(0, n, int(dup.sum()))]
        out[sid] = dict(times=t, cols={"f0": (L.TYPE_FLOAT, rng.normal(100, 20, n), rng.random(n) >= 0.05),
                                       "f1": (L.TYPE_INT, rng.integers(-1000, 1000, n).cumsum(), rng.random(n) >= 0.05),
                                       "f2": (L.TYPE_BOOL, (rng.random(n) < 0.5).astype(np.uint8), rng.random(n) >= 0.05)})
    return out


def flush_timed(sh, desc):
    info = L.RowsInfo()
    t = time.perf_counter()
    L.check(L.lib().og_shard_append_rows(sh.h, desc, info), "og_shard_append_rows")
    ms = (time.perf_counter() - t) * 1e3  # the call synchronises the device before it returns
    return ms, Shard._rows_info(info)


def model_files(batch, last):
    t = time.perf_counter()
    files = fm.files(batch, last)
    descs = [(fm.file_desc(f), ooo) for f, ooo in files]
    return descs, (time.perf_counter() - t) * 1e3


def digest(sh):
    """SHA-256 of the whole export: directory and data region.  Both appends gather the live pages in directory order, so equal
    directories and pages give equal data regions."""
    ex = sh.export()
    h = hashlib.sha256()
    for k in sorted(ex):
        h.update(np.ascontiguousarray(ex[k]))
    return h.hexdigest()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--series", type=int, default=2000)
    ap.add_argument("--rows", type=int, default=1_000_000)
    ap.add_argument("--flush-rows", type=int, default=10_000)
    ap.add_argument("--query-reps", type=int, default=5)
    a = ap.parse_args()
    Shard.init(0)
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    res = dict(card=card, base=f"{a.series} series x {a.rows} float64 rows (G-hi), 1 s cadence, 1000-row segments",
               flushes=f"(a) {a.series} x {a.flush_rows} ordered float rows; (b) {a.series} x {a.flush_rows} rows of float + int + bool, "
                       "5 % nulls, 1 % late inside (a), 5 % repeated times")
    tiny = Shard.synth(a.series, 1, COLS, t0=T0, dt=SEC, seed=1001)
    sids = [int(s) for s in tiny.export()["sids"]]
    tiny.close()
    rng = np.random.default_rng(7)
    ba, bb = batch_a(rng, sids, a.rows, a.flush_rows), batch_b(rng, sids, a.rows, a.flush_rows)
    da, db = Shard.batch_desc(ba), Shard.batch_desc(bb)
    tmax = T0 + (a.rows + 2 * a.flush_rows) * SEC
    # ---- the flushes as rows ----
    sh = Shard.synth(a.series, a.rows, COLS, t0=T0, dt=SEC, seed=1001)
    last_a = {sid: T0 + (a.rows - 1) * SEC for sid in sids}
    res["query_before"] = query_times(sh, tmax, a.query_reps)
    ms_a, info_a = flush_timed(sh, da)
    after_a = query_times(sh, tmax, a.query_reps)
    check_a = (sh.info(), sh.merge_info(), digest(sh))
    last_b = {sid: T0 + (a.rows + a.flush_rows - 1) * SEC for sid in sids}
    ms_b, info_b = flush_timed(sh, db)
    after_b = query_times(sh, tmax, a.query_reps)
    check_b = (sh.info(), sh.merge_info(), digest(sh))
    sh.close()
    L.lib().og_release_cached_memory()
    res["rows_a"] = dict(wall_ms=ms_a, info=info_a, merge_ms=check_a[1]["merge_ms"], after=after_a)
    res["rows_b"] = dict(wall_ms=ms_b, info=info_b, merge_ms=check_b[1]["merge_ms"], after=after_b)
    # ---- the same rows as pre-encoded files on a twin ----
    fa, enc_a = model_files(ba, last_a)
    fb, enc_b = model_files(bb, last_b)
    tw = Shard.synth(a.series, a.rows, COLS, t0=T0, dt=SEC, seed=1001)
    _r, fms_a = timed(lambda: tw.append_files(fa))
    same_a = (tw.info(), tw.merge_info(), digest(tw))
    _r, fms_b = timed(lambda: tw.append_files(fb))
    same_b = (tw.info(), tw.merge_info(), digest(tw))
    tw.close()
    L.lib().og_release_cached_memory()
    for name, got, want in (("a", check_a, same_a), ("b", check_b, same_b)):
        assert got[0] == want[0], (name, got[0], want[0])
        gm, wm = dict(got[1]), dict(want[1])
        gm.pop("merge_ms"); wm.pop("merge_ms")
        assert gm == wm, (name, gm, wm)
        assert got[2] == want[2], f"flush {name}: directory or pages differ from the append_files twin"
    res["files_a"] = dict(wall_ms=fms_a, merge_ms=same_a[1]["merge_ms"], n_files=len(fa),
                          host_encode_ms_oracle_cpp_encoders_per_segment=enc_a)
    res["files_b"] = dict(wall_ms=fms_b, merge_ms=same_b[1]["merge_ms"], n_files=len(fb), merge_info=same_b[1],
                          host_encode_ms_oracle_cpp_encoders_per_segment=enc_b)
    res["answer_check"] = "og_shard_info, og_shard_merge_info, directory and data region (SHA-256 of the export) equal the append_files twin after (a) and (b)"
    # ---- flush (a)'s kernels, in a separate run on a fresh base ----
    from torch.profiler import ProfilerActivity, profile
    sh = Shard.synth(a.series, a.rows, COLS, t0=T0, dt=SEC, seed=1001)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        ms_p, _i = flush_timed(sh, da)
    sh.close()
    ku = kernel_us(prof)
    res["kernels_a_ms"] = {k: v / 1e3 for k, v in sorted(ku.items(), key=lambda kv: -kv[1])[:10]}
    res["kernels_a_total_ms"] = sum(ku.values()) / 1e3
    res["kernels_a_wall_ms_under_profiler"] = ms_p
    print(json.dumps(res))


if __name__ == "__main__":
    main()
