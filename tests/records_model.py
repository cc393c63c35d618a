"""What og_query_next returns for a dense record: a model of TransIntervalRec2Rec slicing (test infrastructure).

KeyCursor.Next hands out a tagset's interval record in slices of ChunkSizeNum windows (agg_tagset_cursor.go:993-1006,
lib/record/record.go:1340-1358).  records_of() restates that over the dense record AggQuery.dense_host() returns;
assert_records() compares what AggQuery.records() drained with it."""
import numpy as np

from opengemini_b200 import _lib as L


def records_of(d, calls, ascending, chunk):
    """what og_query_next returns for dense record d: per tagset, slices of `chunk` windows (latest first when descending)
    without their empty windows; a row's time is the window start (0 without an interval) or, for a single-call selector,
    the selected point's time; multi-call first / last carry RecMeta.Times.  Returns [(group, times, [(valid, value bits,
    times or None) per call])]"""
    nb, multi = d["n_buckets"], len(calls) > 1
    out = []
    for g in range(d["n_groups"]):
        for s in range(0, nb, chunk):
            rows = []
            for b in range(s, min(nb, s + chunk)):
                i = g * nb + (b if ascending else nb - 1 - b)
                if any(c["valid"][i] for c in d["cols"]):
                    rows.append((i, i - g * nb))
            if not rows:
                continue
            times, cols = [], []
            for i, bb in rows:
                t = d["start"] + bb * d["interval"]
                for (f, _c), c in zip(calls, d["cols"]):
                    if c["times"] is not None and not multi and c["valid"][i]:
                        t = int(c["times"][i])
                times.append(t)
            for (f, col), c in zip(calls, d["cols"]):
                idx = np.array([i for i, _ in rows])
                ok = np.asarray(c["valid"])[idx] != 0
                v = np.asarray(c["values"]).view(np.uint64)[idx][ok]
                ct = np.where(ok, np.asarray(c["times"])[idx], 0) if multi and c["times"] is not None else None
                cols.append((ok, v, ct))
            out.append((g, np.array(times, np.int64), cols))
    return out


def assert_records(recs, want, label, sids=None):
    """recs: AggQuery.records() drained; want: records_of().  sids: the shard's sids for per-series output (a record of tagset g
    carries sids[g]), None for tagset maps and one tagset (sid 0)."""
    assert len(recs) == len(want), f"{label}: {len(recs)} records, the model has {len(want)}"
    for n, (r, (g, times, cols)) in enumerate(zip(recs, want)):
        assert r["group"] == g, f"{label} record {n}: group {r['group']}, the model's is {g}"
        assert r["sid"] == (0 if sids is None else int(sids[g])), f"{label} record {n}: sid {r['sid']}"
        assert r["rows"] == times.size and np.array_equal(r["times"], times), f"{label} record {n} (group {g}): row times"
        for k, (rc, (ok, v, ct)) in enumerate(zip(r["cols"], cols)):
            assert np.array_equal(rc["valid"], ok), f"{label} record {n} col {k}: validity"
            assert rc["nil_count"] == int((~ok).sum()), f"{label} record {n} col {k}: nil count"
            rv = rc["values"].astype(np.uint64) if rc["type"] == L.TYPE_BOOL else rc["values"].view(np.uint64)
            assert np.array_equal(rv, v), f"{label} record {n} col {k}: values"
            assert (rc["times"] is None) == (ct is None), f"{label} record {n} col {k}: times presence"
            if ct is not None:
                assert np.array_equal(rc["times"], ct), f"{label} record {n} col {k}: times"
