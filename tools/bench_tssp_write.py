"""og_shard_write_tssp against og_shard_export of the same shard (the device-to-host copy no writer can beat).

Legs (each: one warm-up call, then the median of --reps calls; the host clock runs around calls that return synchronised):
  downsampled   the whole-shard downsample output of tools/bench_downsample_shard.py (125 series x 10^6 rows, 4 float + 2 int +
                1 bool field, 5-minute windows, the per-type policy: 34 columns), reopened in place and written as one file
  big           --big-series x --big-rows float rows (2000 x 10^6: 12 GB of Gorilla pages).  A file holds at most 8 GiB, so the
                shard is written as one file per --big-range series; the times of the ranges are added up
For every leg: write_ms (og_shard_write_tssp: the four phases the library reports, medians of the same calls), image_export_ms
(og_tssp_image_export into a host buffer), shard_export_ms (og_shard_export of the data region into a host buffer), and the
ratio (write + image export) / shard export.  The written file of the first leg is reopened and compared page for page first.

Prints one JSON line; --out also writes it to a file.  Run from the repository root after __graft_entry__.build().
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from opengemini_b200 import Shard, write_tssp  # noqa: E402
from opengemini_b200 import _lib as L  # noqa: E402

T0, SEC = 1_700_000_000_000_000_000, 1_000_000_000
ALL6 = ["min", "max", "sum", "count", "first", "last"]
PHASES = ("preagg", "layout_gather_crc", "metadata_d2h", "host_assembly")


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
        name, power, clock = [x.strip() for x in out.split(",")]
        return dict(gpu=name, power_limit=power, max_sm_clock=clock)
    except Exception as e:
        return dict(gpu=f"unknown ({e})")


def write_once(sh, ranges, host):
    """One file per series range: (write ms, export ms, phase ms, total file bytes)."""
    lib = L.lib()
    w_ms = e_ms = 0.0
    ph = np.zeros(4)
    total = 0
    for r in ranges:
        d = L.TsspWriteDesc(b"bench", r[0], r[1], 0)
        h = C.c_void_p()
        t = time.perf_counter()
        L.check(lib.og_shard_write_tssp(sh.h, C.byref(d), C.byref(h)), "og_shard_write_tssp")   # returns synchronised
        w_ms += (time.perf_counter() - t) * 1e3
        n = C.c_uint64()
        L.check(lib.og_tssp_image_size(h, C.byref(n)), "og_tssp_image_size")
        assert n.value <= host.size
        t = time.perf_counter()
        L.check(lib.og_tssp_image_export(h, host.ctypes.data), "og_tssp_image_export")          # a blocking copy
        e_ms += (time.perf_counter() - t) * 1e3
        ms = (C.c_double * 4)()
        L.check(lib.og_tssp_image_timing(h, ms), "og_tssp_image_timing")
        ph += np.array(list(ms))
        total += n.value
        lib.og_tssp_image_free(h)
    return w_ms, e_ms, ph, total


def leg(sh, ranges, reps):
    lay = L.ShardLayout()
    L.check(L.lib().og_shard_layout_get(sh.h, C.byref(lay)), "og_shard_layout_get")
    host = np.empty(lay.data_len + (64 << 20), np.uint8)   # a file is smaller than the data region plus its directory
    host[:] = 0                                            # touch the pages before anything is timed

    def shard_export():
        t = time.perf_counter()
        L.check(L.lib().og_shard_export(sh.h, host.ctypes.data, None, None, None, None, None, None, None), "og_shard_export")
        return (time.perf_counter() - t) * 1e3

    write_once(sh, ranges, host)
    shard_export()
    w, e, ph, x = [], [], [], []
    for _ in range(reps):                                  # the two sides alternate
        wm, em, p, total = write_once(sh, ranges, host)
        w.append(wm); e.append(em); ph.append(p)
        x.append(shard_export())
    wm, em, xm = float(np.median(w)), float(np.median(e)), float(np.median(x))
    phm = np.median(np.array(ph), axis=0)
    info = sh.info()
    return dict(series=info["n_series"], segments=info["n_segments"], rows=info["n_rows"], columns=lay.n_columns, files=len(ranges),
                shard_data_bytes=lay.data_len, file_bytes=total, write_ms=round(wm, 3), image_export_ms=round(em, 3),
                shard_export_ms=round(xm, 3), phases_ms_median={k: round(float(v), 3) for k, v in zip(PHASES, phm)},
                write_plus_export_over_shard_export=round((wm + em) / xm, 3),
                shard_export_GBps=round(lay.data_len / xm / 1e6, 2), image_export_GBps=round(total / em / 1e6, 2))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--series", type=int, default=125)
    ap.add_argument("--rows", type=int, default=1_000_000)
    ap.add_argument("--interval-s", type=int, default=300)
    ap.add_argument("--big-series", type=int, default=2000)
    ap.add_argument("--big-rows", type=int, default=1_000_000)
    ap.add_argument("--big-range", type=int, default=1000)
    ap.add_argument("--reps", type=int, default=9)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    Shard.init(0)
    res = dict(workload="tssp_write", reps=a.reps, **gpu_info())

    cols = [(L.TYPE_FLOAT, L.SYNTH_F_HI, 0), (L.TYPE_FLOAT, L.SYNTH_F_LO, 0), (L.TYPE_FLOAT, L.SYNTH_F_HI, 0), (L.TYPE_FLOAT, L.SYNTH_F_LO, 0),
            (L.TYPE_INT, L.SYNTH_INT_WALK, 0), (L.TYPE_INT, L.SYNTH_INT_WALK, 0), (L.TYPE_BOOL, L.SYNTH_BOOL, 0)]
    src = Shard.synth(a.series, a.rows, cols, t0=T0, dt=SEC, seed=4)
    ds = src.downsample_shard(a.interval_s * SEC, T0, T0 + (a.rows - 1) * SEC,
                              {L.TYPE_FLOAT: ALL6, L.TYPE_INT: ["min", "max", "sum", "count"], L.TYPE_BOOL: ["count", "last"]})
    new = ds.open()
    back = Shard.open_tssp(write_tssp(new, "bench"))
    ea, eb = new.export(), back.export()
    for c in range(ea["page_off"].shape[0]):
        assert np.array_equal(ea["page_len"][c], eb["page_len"][c])
        for g in range(ea["page_len"].shape[1]):
            assert ea["data"][int(ea["page_off"][c, g]):int(ea["page_off"][c, g]) + int(ea["page_len"][c, g])].tobytes() == \
                eb["data"][int(eb["page_off"][c, g]):int(eb["page_off"][c, g]) + int(eb["page_len"][c, g])].tobytes(), (c, g)
    back.close()
    res["downsampled"] = leg(new, [(0, 0)], a.reps)
    new.close(); ds.close(); src.close()

    if a.big_series:
        big = Shard.synth(a.big_series, a.big_rows, [(L.TYPE_FLOAT, L.SYNTH_F_HI, 0)], t0=T0, dt=SEC, seed=4)
        ranges = [(b, min(a.big_series, b + a.big_range)) for b in range(0, a.big_series, a.big_range)]
        res["big"] = leg(big, ranges, a.reps)
        big.close()
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
