"""Whole-shard downsample (og_downsample_shard) at the configs[4] shape: one shard of 125 series x 10^6 rows at a 1 s cadence
with 4 float, 2 int and 1 bool field, 5-minute windows.

Legs, run one after the other (each timed as the median of --reps calls after one warm-up call; every call returns
synchronised; phase times are the medians of the same calls):
  policy      a per-type policy: float {min,max,sum,count,first,last}, int {min,max,sum,count}, bool {count,last}
              -> rows/s of the source rows in range, and the phase times the library reports (og_downsampled_timing)
  six_shard   float and int fields with all six calls, one og_downsample_shard call
  six_percol  the same output from one og_downsample call per float / int field, stitched into one shard: the data regions
              concatenated on the device, the directories on the host.  (The shard has no nulls, so every field keeps the same
              windows and a plain stitch is exact; og_downsample refuses bool fields, so they are not in either six-call leg.)
The six-call legs are checked page for page against each other before anything is timed.

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

from opengemini_b200 import Shard  # noqa: E402
from opengemini_b200 import _lib as L  # noqa: E402
from opengemini_b200.cursor import device_view  # noqa: E402

T0, SEC = 1_700_000_000_000_000_000, 1_000_000_000
ALL6 = ["min", "max", "sum", "count", "first", "last"]


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
        name, power, clock = [x.strip() for x in out.split(",")]
        return dict(gpu=name, power_limit=power, max_sm_clock=clock)
    except Exception as e:  # the numbers are still reported; say where they came from is unknown
        return dict(gpu=f"unknown ({e})")


def timed(fn, reps):
    """Median wall time of `reps` calls after a warm-up, the last result, and the median of each phase og_downsampled_timing
    reports (when the result has them)."""
    fn().close()  # warm-up
    ts, phases, last = [], [], None
    for _ in range(reps):
        if last is not None:
            last.close()
        t = time.perf_counter()
        last = fn()
        ts.append((time.perf_counter() - t) * 1e3)
        if hasattr(last, "timing"):
            phases.append(last.timing())
    med = {k: round(float(np.median([p[k] for p in phases])), 3) for k in phases[0]} if phases else None
    return float(np.median(ts)), last, med


class Stitched:
    """Per-column og_downsample results stitched into one shard: device data concatenated, directories merged on the host."""

    def __init__(self, parts, torch):
        self.parts = parts
        blobs, pos, self.columns = [], 0, []
        for k, p in enumerate(parts):
            d = p.desc
            blobs.append(device_view(C.cast(d.data, C.c_void_p).value, d.data_len, "|u1", torch.device("cuda", 0)))
            cols, (tpo, tpl) = p.columns()
            for name, typ, po, pl in cols:
                self.columns.append((name, typ, po + np.uint64(pos), pl))
            if k == 0:
                self.time = (tpo.copy(), tpl.copy())
                ns = d.n_series
                self.ssb = np.ctypeslib.as_array(d.series_seg_begin, shape=(ns + 1,)).copy()
            pos += d.data_len
        self.columns.sort(key=lambda c: c[0])
        self.data = torch.cat(blobs + [torch.zeros(1024, dtype=torch.uint8, device=blobs[0].device)])
        torch.cuda.synchronize()
        self.data_len = pos

    def close(self):
        for p in self.parts:
            p.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--series", type=int, default=125)
    ap.add_argument("--rows", type=int, default=1_000_000)
    ap.add_argument("--interval-s", type=int, default=300)
    ap.add_argument("--reps", type=int, default=9)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch

    Shard.init(0)
    cols = [(L.TYPE_FLOAT, L.SYNTH_F_HI, 0), (L.TYPE_FLOAT, L.SYNTH_F_LO, 0), (L.TYPE_FLOAT, L.SYNTH_F_HI, 0), (L.TYPE_FLOAT, L.SYNTH_F_LO, 0),
            (L.TYPE_INT, L.SYNTH_INT_WALK, 0), (L.TYPE_INT, L.SYNTH_INT_WALK, 0), (L.TYPE_BOOL, L.SYNTH_BOOL, 0)]
    sh = Shard.synth(a.series, a.rows, cols, t0=T0, dt=SEC, seed=4)
    ivl, tmin, tmax = a.interval_s * SEC, T0, T0 + (a.rows - 1) * SEC
    src_rows = a.series * a.rows
    policy = {L.TYPE_FLOAT: ALL6, L.TYPE_INT: ["min", "max", "sum", "count"], L.TYPE_BOOL: ["count", "last"]}
    six = {L.TYPE_FLOAT: ALL6, L.TYPE_INT: ALL6}
    numeric = [c for c, (t, _d, _n) in enumerate(cols) if t in (L.TYPE_FLOAT, L.TYPE_INT)]

    # the two six-call legs produce the same shard
    ref = Stitched([sh.downsample(c, ivl, tmin, tmax) for c in numeric], torch)
    got = sh.downsample_shard(ivl, tmin, tmax, six)
    gcols, (gtpo, gtpl) = got.columns()
    gdata, rdata = got.export(), ref.data[:ref.data_len].cpu().numpy()
    assert [c[0] for c in gcols] == [c[0] for c in ref.columns], "column names differ"
    assert np.array_equal(np.ctypeslib.as_array(got.desc.series_seg_begin, shape=(a.series + 1,)), ref.ssb)
    for (name, _t, po, pl), (_n, _rt, rpo, rpl) in zip(gcols + [("time", 0, gtpo, gtpl)], ref.columns + [("time", 0, *ref.time)]):
        assert np.array_equal(pl, rpl), name
        for g in range(po.size):
            assert gdata[po[g]:po[g] + pl[g]].tobytes() == rdata[rpo[g]:rpo[g] + rpl[g]].tobytes(), (name, g)
    n_checked = len(gcols)
    got.close(); ref.close()

    res = dict(workload="downsample_shard", series=a.series, rows_per_series=a.rows, fields="4 float, 2 int, 1 bool",
               interval_s=a.interval_s, source_rows=src_rows, reps=a.reps, **gpu_info())
    ms, out, ph = timed(lambda: sh.downsample_shard(ivl, tmin, tmax, policy), a.reps)
    res["policy"] = dict(ms=round(ms, 3), rows_per_s=src_rows / (ms / 1e3), out_columns=out.desc.n_columns, out_rows=out.rows,
                         out_segments=out.desc.n_segments, out_bytes=out.desc.data_len,
                         phases_ms_median=ph)
    out.close()
    ms, out, ph = timed(lambda: sh.downsample_shard(ivl, tmin, tmax, six), a.reps)
    res["six_shard"] = dict(ms=round(ms, 3), rows_per_s=src_rows / (ms / 1e3), out_columns=out.desc.n_columns, phases_ms_median=ph)
    out.close()
    ms, out, _ = timed(lambda: Stitched([sh.downsample(c, ivl, tmin, tmax) for c in numeric], torch), a.reps)
    res["six_percol"] = dict(ms=round(ms, 3), rows_per_s=src_rows / (ms / 1e3), out_columns=len(out.columns),
                             pages_checked_equal_columns=n_checked)
    out.close()
    sh.close()
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
