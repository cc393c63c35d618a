"""A wide aggregate: count and sum over six columns with a two-term WHERE, the shape that k_fused_cols does not take.

    python tools/bench_wide.py [--series 10000] [--rows 10000] [--reps 5] [--runs 3] [--lib NAME=PATH ...] [--out DIR]

Shard: og_shard_synth, 1 s cadence, 1000-row segments, three float64 columns (G-hi, G-lo, G-hi with 5 % nulls), two int64
columns (random walks, one with 2 % nulls) and one bool column.  Query: eight calls (the most a query takes), sum of every
numeric column and count of the bool and of the two columns with nulls, GROUP BY time(1m), WHERE f0 > 100.5 AND i0 < 0, one
tagset.  It runs on og_stats.path 0, the materialise-tile path, which serves queries over more than 4 columns that
k_fused_cols does not take.

Each --lib is a build of libogpu.so (default: the in-tree one).  The libraries run alternately, each in a process of its own
(the library is chosen at import through OGPU_LIB), `--runs` times each; a process builds the shard, runs the query once to
warm up and then `--reps` times.  Prints one JSON line per process (og_stats.main_kernel_ms and kernel_ms as the median over
the reps, G rows/s from the median kernel_ms, og_stats.path) and a last line with the card, its power limit and whether the
dense outputs of all libraries are bitwise equal.  With --out the dense outputs go to DIR as .npz files; without it to a
temporary directory.  Needs a GPU.
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
T0, SEC = 1_700_000_000_000_000_000, 1_000_000_000


def worker(a):
    sys.path.insert(0, ROOT)
    from opengemini_b200 import AggQuery, Shard
    from opengemini_b200 import _lib as L
    Shard.init(0)
    cols = [(L.TYPE_FLOAT, L.SYNTH_F_HI, 0), (L.TYPE_FLOAT, L.SYNTH_F_LO, 0), (L.TYPE_FLOAT, L.SYNTH_F_HI, 50),
            (L.TYPE_INT, L.SYNTH_INT_WALK, 0), (L.TYPE_INT, L.SYNTH_INT_WALK, 20), (L.TYPE_BOOL, L.SYNTH_BOOL, 0)]
    sh = Shard.synth(a.series, a.rows, cols, t0=T0, dt=SEC, seed=17)
    calls = [("sum", c) for c in range(5)] + [("count", 5), ("count", 2), ("count", 4)]
    flt = [("term", 0, ">", 100.5), ("term", 3, "<", 0), "and"]
    q = AggQuery(sh, calls, 60 * SEC, T0, T0 + (a.rows - 1) * SEC, filter=flt)
    q.run()  # warm-up: plan, scratch, module load
    main, total = [], []
    for _ in range(a.reps):
        st = q.run().stats()
        main.append(st["main_kernel_ms"]); total.append(st["kernel_ms"])
    d = q.dense_host()
    np.savez(a.worker_out, **{f"{k}_{i}": c[k] for i, c in enumerate(d["cols"]) for k in ("values", "valid") if c[k] is not None})
    kms = float(np.median(total))
    print(json.dumps(dict(lib=a.name, path=st["path"], main_kernel_ms=round(float(np.median(main)), 3), kernel_ms=round(kms, 3),
                          g_rows_per_s=round(st["rows_decoded"] / kms / 1e6, 2), rows=st["rows_decoded"], page_bytes=st["page_bytes"],
                          calls=len(calls))), flush=True)
    q.close()
    sh.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--series", type=int, default=10000)
    ap.add_argument("--rows", type=int, default=10000)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--lib", action="append", default=[], help="NAME=PATH of a libogpu.so build")
    ap.add_argument("--out")
    ap.add_argument("--worker", action="store_true", help=argparse.SUPPRESS)
    ap.add_argument("--name", help=argparse.SUPPRESS)
    ap.add_argument("--worker-out", help=argparse.SUPPRESS)
    a = ap.parse_args()
    if a.worker:
        return worker(a)
    libs = [tuple(s.split("=", 1)) for s in a.lib] or [("tree", os.path.join(ROOT, "opengemini_b200", "libogpu.so"))]
    with tempfile.TemporaryDirectory() as tmp:
        out = a.out or tmp
        os.makedirs(out, exist_ok=True)
        for r in range(a.runs):
            for name, path in libs:
                env = dict(os.environ, OGPU_LIB=os.path.abspath(path))
                subprocess.run([sys.executable, os.path.abspath(__file__), "--worker", "--name", name, "--series", str(a.series),
                                "--rows", str(a.rows), "--reps", str(a.reps), "--worker-out", os.path.join(out, f"{name}_{r}.npz")],
                               env=env, check=True)
        ref = np.load(os.path.join(out, f"{libs[0][0]}_0.npz"))
        same = {}
        for name, _ in libs:
            for r in range(a.runs):
                got = np.load(os.path.join(out, f"{name}_{r}.npz"))
                same[f"{name}_{r}"] = sorted(got.files) == sorted(ref.files) and all(np.array_equal(got[k], ref[k]) for k in ref.files)
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    print(json.dumps(dict(gpu=gpu, series=a.series, rows=a.rows, bitwise_equal_to_first=same)))


if __name__ == "__main__":
    main()
