"""The cross-shard merge on float, int and bool columns: og_query_merge_dense (k_merge_dense) and og_query_allreduce
(k_merge_pack -> NCCL -> k_merge_unpack), on every call alone, mixed call sets, tagset maps, ties, NaN, signed zeros, integer
sums that wrap, empty shards and fields, a chain of three shards, and the records read after a merge.

Every shard has one schema: F, a float column (36-bit-mantissa values in [100, 101) with a share of 99.5 / 101.5, so extremes
tie across series and shards), I, an int column (a Simple8b random walk with a share of -+10^7, the same), and B, a bool column.
Every series ticks on one 1 s cadence, so first / last tie on time across all series of all shards.  Sids differ across shards.

Each test names the shards it merges (A <- B: B merged into A, A <- B <- C for a chain) and the combined shard the oracle
scans: the series of A, then B, then C, in one shard, with the tagset maps concatenated the same way -- the reference's
cross-series update order (lib/record/reccord_functions.go).  Against that scan everything is bitwise: values, validity and the
time of every selector.  Float sums are not (the merge adds whole shards' partial sums); they get two checks instead:

  exact association   the merged cell is, bit for bit, the float64 sum of the per-shard oracle cells in the order the merge adds
                      them -- group_update adds p + a, so B + A, and C + (B + A) for a chain (an empty side adds 0.0).  A window
                      holding NaN or an infinity is NaN on both sides (payload not compared), or the same infinity;
  high precision      on finite windows, within n * 2^-53 * sum|x| of math.fsum over the window's rows of all shards
                      (segment_shards.window_model; n the window's row count).

NaN makes the reference's own update depend on the order of the partials: a cell holding NaN is replaced by the next partial
(every comparison with NaN is false).  Merging whole shards therefore equals the combined scan only when the NaN rows lie in the
shard merged into -- its fold is the combined scan's prefix -- and the NaN cases put them there.
"""
import ctypes as C
import os
import tempfile

import numpy as np
import pytest

import oracle
import segment_shards as ss
from opengemini_b200 import AggQuery, Comm, Shard
from opengemini_b200 import _lib as L
from records_model import assert_records, records_of

pytestmark = pytest.mark.gpu

T0, SEC = ss.T0, ss.SEC
KINDS = ["f_hi", "i_s8b", "bool"]
TYPES = ss.types_of(KINDS)
F, I, B = range(3)
ALL6 = ["count", "sum", "min", "max", "first", "last"]
FUNCS = {F: ALL6, I: ALL6, B: [f for f in ALL6 if f != "sum"]}  # sum() of a bool column is refused at create
SINGLE = [[(f, c)] for c in (F, I, B) for f in FUNCS[c]]
MIXED8 = [("sum", F), ("sum", I), ("count", B), ("min", I), ("max", F), ("first", B), ("last", I), ("count", F)]
MIXED = [MIXED8,
         [("min", F), ("max", F)],                            # two calls: min / max carry no time
         [("min", I), ("max", B)],
         [("first", F), ("last", F), ("first", I), ("last", B), ("count", I)],  # RecMeta.Times of several columns
         [("sum", I), ("count", B), ("sum", F)]]
NG = 3
SELECTORS = ("min", "max", "first", "last")


@pytest.fixture(scope="module", autouse=True)
def _device():
    Shard.init(0)


# ---------------------------------------------------------------------------------------------------------------
# shards
# ---------------------------------------------------------------------------------------------------------------
def _desc(pieces):
    """host shard desc of the series of `pieces`, in order; a column a piece never wrote gets page_len 0 in its segments"""
    d = ss.shard_desc([s for p in pieces for s in p.series], TYPES, [x for p in pieces for x in p.lengths],
                      np.concatenate([p.sids for p in pieces]))
    seg0 = 0
    for p in pieces:
        nseg = sum(len(x) for x in p.lengths)
        for c in p.absent:
            np.ctypeslib.as_array(d.columns[c].page_len, shape=(d.n_segments,))[seg0:seg0 + nseg] = 0
        seg0 += nseg
    return d


class Piece:
    """One shard: per-series rows (segment_shards.series_rows), the segment lengths of each series, their sids and tagsets.
    absent: columns the shard never wrote (every row null, page_len 0 in every segment)."""

    def __init__(self, series, lengths, sid0, groups=None, absent=()):
        self.series, self.lengths, self.absent = series, lengths, tuple(absent)
        for c in self.absent:
            for s in series:
                s["cols"][c] = (s["cols"][c][0], np.zeros(s["times"].size, bool))
        self.sids = np.arange(sid0, sid0 + len(series), dtype=np.uint64)
        self.groups = np.zeros(len(series), np.uint32) if groups is None else np.asarray(groups, np.uint32)
        self.sd = _desc([self])
        self.sh = Shard.open_desc(self.sd, keepalive=self.sd)

    def close(self):
        self.sh.close()


def _rows(rng, n, t0=T0, nulls=0.0, ties=0.05):
    r = ss.series_rows(rng, n, KINDS, nulls, t0=t0)
    f, i = r["cols"][F][0], r["cols"][I][0]
    pick = rng.random(n) < ties
    f[pick] = rng.choice([99.5, 101.5], int(pick.sum()))
    pick = rng.random(n) < ties
    i[pick] = rng.choice([-10**7, 10**7], int(pick.sum()))
    return r


def _piece(seed, n_series, rows, sid0, t0=T0, nulls=0.0, cuts=([1000],), groups=None, absent=(), edit=None):
    """edit(series index, rows): change a series' values before its pages are encoded"""
    rng = np.random.default_rng(seed)
    series = [_rows(rng, rows, t0, nulls) for _ in range(n_series)]
    for k, s in enumerate(series):
        if edit:
            edit(k, s)
    return Piece(series, [ss.mixed(cuts[k % len(cuts)], rows) for k in range(n_series)], sid0, groups, absent)


NULLS = [0.05, 0.1, 0.3]


# ---------------------------------------------------------------------------------------------------------------
# queries, merges and checks
# ---------------------------------------------------------------------------------------------------------------
def _query(p, calls, iv, tmin, tmax, offset=0, mapped=False, run=True, **kw):
    if mapped:
        kw.update(group="map", series_group=p.groups, n_groups=NG)
    q = AggQuery(p.sh, calls, iv, tmin, tmax, offset=offset, flags=L.Q_QUERY_GRID | L.Q_STRICT_ORDER, **kw)
    return q.run() if run else q


def _merge(q, other):
    L.check(L.lib().og_query_merge_dense(q.h, C.byref(other.dense_view())), "og_query_merge_dense")


def _oracle(pieces, desc, mapped, sd=None):
    """oracle.scan of the combined shard of `pieces` with `desc`, whose series_group points at the concatenated tagset maps"""
    d = L.QueryDesc.from_buffer_copy(desc)
    if mapped:
        sg = np.ascontiguousarray(np.concatenate([p.groups for p in pieces]), np.uint32)
        d.series_group = sg.ctypes.data_as(C.POINTER(C.c_uint32))
    return oracle.scan(sd if sd is not None else _desc(pieces), d, threads=1)


def _on_grid(part, start, n_buckets):
    """an oracle record laid over the query's grid: the oracle lays a shard's record over the query range cut to the shard's
    own rows, as the reference does without a common grid (OG_Q_QUERY_GRID)"""
    off = (part["start"] - start) // part["interval"] if part["interval"] else 0
    nb, ng = part["n_buckets"], part["n_groups"]
    if (off, nb) == (0, n_buckets):
        return part
    assert 0 <= off and off + nb <= n_buckets, (part["start"], nb, start, n_buckets)
    cols = []
    for c in part["cols"]:
        out = {}
        for name, a in c.items():
            x = np.zeros((ng, n_buckets), a.dtype)
            x[:, off:off + nb] = a.reshape(ng, nb)
            out[name] = x.ravel()
        cols.append(out)
    return dict(part, start=start, n_buckets=n_buckets, cols=cols)


def _sum_as_merged(parts, k):
    """column k's float sums as the merge adds the per-shard cells: B + A, then C + (B + A) (an empty cell adds 0.0)"""
    acc = np.where(parts[0]["cols"][k]["valid"] != 0, parts[0]["cols"][k]["values"].view(np.float64), 0.0)
    for p in parts[1:]:
        acc = np.where(p["cols"][k]["valid"] != 0, p["cols"][k]["values"].view(np.float64) + acc, acc)
    return acc


def _check(got, pieces, descs, calls, q, label, mapped=False, sd=None):
    """got: the merged record (dense_host() form) of `pieces` merged in order; descs: each piece's query descriptor;
    q: (interval, offset, tmin, tmax).  Everything bitwise against the oracle's scan of the combined shard; float sums by
    exact association of the per-shard oracle cells and within n * 2^-53 * sum|x| of the exact sum."""
    ref = _oracle(pieces, descs[0], mapped, sd)
    parts = [_on_grid(oracle.scan(p.sd, d, threads=1), got["start"], got["n_buckets"]) for p, d in zip(pieces, descs)]
    assert (got["n_groups"], got["n_buckets"], got["start"]) == (ref["n_groups"], ref["n_buckets"], ref["start"]), label
    multi = len(calls) > 1
    for k, (f, col) in enumerate(calls):
        g, r = got["cols"][k], ref["cols"][k]
        ok = r["valid"] != 0
        where = f"{label} call {k} {f}({KINDS[col]})"
        assert np.array_equal(np.asarray(g["valid"]) != 0, ok), f"{where}: validity differs at {np.flatnonzero((np.asarray(g['valid']) != 0) != ok)[:5]}"
        gu = np.asarray(g["values"]).view(np.uint64)
        if f == "sum" and TYPES[col] == L.TYPE_FLOAT:
            want, gf = _sum_as_merged(parts, k), gu.view(np.float64)
            same = (gu == want.view(np.uint64)) | (np.isnan(gf) & np.isnan(want))
            assert same[ok].all(), f"{where}: {int((~same[ok]).sum())} cells are not the float64 sum of the shards' cells in merge order"
            iv, off, tmin, tmax = q
            groups = np.concatenate([p.groups for p in pieces]) if mapped else np.zeros(sum(len(p.series) for p in pieces), int)
            m = ss.window_model([s for p in pieces for s in p.series], col, L.TYPE_FLOAT, iv, off, tmin, tmax, groups)
            assert m["count"].size == ok.size and np.array_equal(m["valid"], ok), f"{where}: model geometry"
            fin = ok & np.isfinite(m["sum_exact"]) & np.isfinite(m["sum_abs"])
            err = np.abs(gf - m["sum_exact"])
            assert np.all(err[fin] <= (m["count"] * 2.0**-53 * m["sum_abs"])[fin]), f"{where}: beyond n*2^-53*sum|x| of the exact sum"
            continue
        bad = np.flatnonzero(gu[ok] != r["values"][ok])
        assert bad.size == 0, f"{where}: {bad.size} value cells differ, first gpu={gu[ok][bad[:3]]} ref={r['values'][ok][bad[:3]]}"
        if f in SELECTORS and not (multi and f in ("min", "max")):
            assert g["times"] is not None, f"{where}: no times"
            assert np.array_equal(np.asarray(g["times"])[ok], r["times"][ok]), f"{where}: selector times differ"


def _merged(pieces, calls, q, label, mapped=False, sd=None):
    """run `calls` on every piece, merge them into the first in order (A <- B <- C), check the merged record; returns it"""
    iv, off, tmin, tmax = q
    qs = [_query(p, calls, iv, tmin, tmax, off, mapped) for p in pieces]
    try:
        for other in qs[1:]:
            _merge(qs[0], other)
        got = qs[0].dense_host()
        _check(got, pieces, [x.desc for x in qs], calls, q, label, mapped, sd)
        return got
    finally:
        for x in qs:
            x.close()


def _same(got, want, label):
    """two records bitwise: validity, and values and selector times on the valid cells"""
    assert (got["n_groups"], got["n_buckets"], got["start"]) == (want["n_groups"], want["n_buckets"], want["start"]), label
    for k, (g, w) in enumerate(zip(got["cols"], want["cols"])):
        ok = np.asarray(w["valid"]) != 0
        assert np.array_equal(np.asarray(g["valid"]) != 0, ok), f"{label} call {k}: validity"
        assert np.array_equal(np.asarray(g["values"]).view(np.uint64)[ok], np.asarray(w["values"]).view(np.uint64)[ok]), f"{label} call {k}: values"
        assert (g["times"] is None) == (w["times"] is None), f"{label} call {k}: times presence"
        if w["times"] is not None:
            assert np.array_equal(np.asarray(g["times"])[ok], np.asarray(w["times"])[ok]), f"{label} call {k}: times"


def _span(pieces):
    return int(min(s["times"][0] for p in pieces for s in p.series)), int(max(s["times"][-1] for p in pieces for s in p.series))


def _grid_queries(tmin, tmax):
    """(interval, offset, tmin, tmax): 60 s, 7 s, no interval, and 60 s windows offset by 13 s over a range cut inside segments"""
    span = tmax - tmin
    return [(60 * SEC, 0, tmin, tmax), (7 * SEC, 0, tmin, tmax), (0, 0, tmin, tmax),
            (60 * SEC, 13 * SEC, tmin + span // 4 + 7, tmax - span // 6)]


def _pair(shifted, nulls=0.0, mapped=False, rows=2400):
    """A: 5 series cut in 1000-row and 333/1000-row segments; B: 4 series of 700 and 1000/31 rows, sharing A's range or
    starting 1700 s later"""
    a = _piece(1, 5, rows, 1, nulls=nulls, cuts=([1000], [333, 1000]), groups=[0, 1, 2, 0, 1] if mapped else None)
    b = _piece(2, 4, rows, 101, t0=T0 + (1700 * SEC if shifted else 0), nulls=nulls, cuts=([700], [1000, 31]),
               groups=[2, 2, 0, 0] if mapped else None)
    return a, b


# ---------------------------------------------------------------------------------------------------------------
# og_query_merge_dense
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("shifted", [False, True], ids=["same-range", "shifted-range"])
def test_every_call_alone_on_every_type(shifted):
    """A <- B; the oracle scans [A's series, B's series]; float sums: B + A"""
    a, b = _pair(shifted)
    sd = _desc([a, b])
    for q in _grid_queries(*_span([a, b])):
        for calls in SINGLE:
            _merged([a, b], calls, q, f"{calls} iv={q[0]} off={q[1]}", sd=sd)
    a.close(); b.close()


@pytest.mark.parametrize("shifted", [False, True], ids=["same-range", "shifted-range"])
def test_mixed_call_sets_across_types(shifted):
    """A <- B with nulls in every column (5 % F, 10 % I, 30 % B); the oracle scans [A, B]; float sums: B + A"""
    a, b = _pair(shifted, NULLS)
    sd = _desc([a, b])
    for q in _grid_queries(*_span([a, b])):
        for calls in MIXED:
            _merged([a, b], calls, q, f"{calls} iv={q[0]} off={q[1]}", sd=sd)
    a.close(); b.close()


def test_tagset_map_with_a_group_empty_in_one_shard():
    """A <- B under OG_GROUP_MAP with three tagsets: A's series in groups [0, 1, 2, 0, 1], B's in [2, 2, 0, 0] (group 1 empty in
    B).  The oracle scans [A, B] with the map [0, 1, 2, 0, 1, 2, 2, 0, 0]; float sums: B + A"""
    a, b = _pair(True, NULLS, mapped=True)
    sd = _desc([a, b])
    lo, hi = _span([a, b])
    for q in [(60 * SEC, 0, lo, hi), (0, 0, lo, hi), (60 * SEC, 13 * SEC, lo + 611 * SEC, hi - 397 * SEC)]:
        for calls in MIXED + SINGLE:
            got = _merged([a, b], calls, q, f"map {calls} iv={q[0]}", mapped=True, sd=sd)
            assert (np.asarray(got["cols"][0]["valid"]).reshape(NG, -1) != 0).any(axis=1).all(), "every tagset holds rows"
    a.close(); b.close()


def _window_edges(t):
    """rows of series times t that are the first and the last of their 60 s window"""
    s = (t // SEC) % 60
    first, last = s == 0, s == 59
    first[0] = last[-1] = True
    return first, last


def test_tied_extremes_across_shards():
    """A <- B over one range.  Every series of both shards holds F = 250.0 / -250.0 and I = +-10^8 at one shared row in 97 (the
    same time in every series) and at one row in 89 / 83 placed by its series (other times); bool extremes tie everywhere.
    min / max keep the earliest time and, at the same time, A's cell; first / last at the shared window edges keep the larger
    value.  The oracle scans [A, B]; float sums: B + A"""
    def extremes(k, s):
        f, i = s["cols"][F][0], s["cols"][I][0]
        f[3::97] = 250.0; f[k % 89::89] = 250.0; f[50::97] = -250.0; f[(5 * k) % 83::83] = -250.0
        i[3::97] = 10**8; i[k % 89::89] = 10**8; i[50::97] = -10**8; i[(5 * k) % 83::83] = -10**8
    a = _piece(11, 5, 2400, 1, cuts=([1000], [333, 1000]), edit=extremes)
    b = _piece(12, 4, 2400, 101, cuts=([700], [1000, 31]), edit=lambda k, s: extremes(k + 2, s))
    sd = _desc([a, b])
    lo, hi = _span([a, b])
    won = {}
    for q in [(60 * SEC, 0, lo, hi), (7 * SEC, 0, lo, hi), (0, 0, lo, hi)]:
        for calls in SINGLE + MIXED:
            got = _merged([a, b], calls, q, f"ties {calls} iv={q[0]}", sd=sd)
            if len(calls) == 1 and calls[0][0] in ("first", "last") and q[0] == 60 * SEC:
                qa = _query(a, calls, q[0], q[2], q[3], q[1])
                own = qa.dense_host()["cols"][0]
                qa.close()
                ok = np.asarray(own["valid"]) != 0
                from_b = np.asarray(got["cols"][0]["values"]).view(np.uint64)[ok] != np.asarray(own["values"]).view(np.uint64)[ok]
                won[calls[0]] = (from_b.any(), (~from_b).any())
    # the equal-time rule decided cells both ways: some windows' first / last come from B's series, some from A's
    for (f, c), (b_won, a_won) in won.items():
        if TYPES[c] != L.TYPE_BOOL:
            assert b_won and a_won, (f, KINDS[c], b_won, a_won)
    a.close(); b.close()


def test_signed_zeros_across_shards():
    """A <- B over one range with F in [0, 1): A holds +0.0 where B holds -0.0, at the first and last row of every 60 s window
    (the same time in every series), at one row in 61 and at one row in 53 placed by the series.  Those zeros are every window's
    minimum, first and last value: each tie keeps A's +0.0 (the cell merged into), and -0.0 only where B's zero is alone or
    earlier.  The oracle scans [A, B]; float sums: B + A"""
    def zeros(z):
        def edit(k, s):
            f = s["cols"][F][0]
            f[:] = np.abs(f - 100.0)
            first, last = _window_edges(s["times"])
            f[first | last] = z
            f[3::61] = z; f[k % 53::53] = z
        return edit
    a = _piece(21, 5, 2400, 1, cuts=([1000], [333, 1000]), edit=zeros(0.0))
    b = _piece(22, 4, 2400, 101, cuts=([700], [1000, 31]), edit=zeros(-0.0))
    sd = _desc([a, b])
    lo, hi = _span([a, b])
    for q in [(60 * SEC, 0, lo, hi), (7 * SEC, 0, lo, hi), (0, 0, lo, hi)]:
        for calls in [[(f, F)] for f in ALL6] + [[("min", F), ("max", F)], [("first", F), ("last", F), ("min", F), ("sum", F)]]:
            got = _merged([a, b], calls, q, f"zeros {calls} iv={q[0]}", sd=sd)
            for k, (f, _c) in enumerate(calls):
                if f in ("first", "last", "min") and q[0] == 60 * SEC:  # the tie of +0.0 and -0.0 happened, and A's zero kept it
                    v = np.asarray(got["cols"][k]["values"]).view(np.float64)[np.asarray(got["cols"][k]["valid"]) != 0]
                    assert np.all(v == 0) and not np.signbit(v).any(), f"{calls} call {k}"
    a.close(); b.close()


def test_nan_rows_in_the_shard_merged_into():
    """A <- B and A <- B <- C, NaN rows only in A (see the module doc): 2 % of A's F rows, and every series' first row of every
    60 s window in one series in two.  A's series are cut in segments of 3, 4 and 1000 rows (raw pages with NaN) or 1000 rows
    (Snappy pages).  The oracle scans [A, B] / [A, B, C]; float sums: B + A, C + (B + A); a window with NaN is NaN in both."""
    def nans(k, s):
        f = s["cols"][F][0]
        f[np.random.default_rng(k).random(f.size) < 0.02] = np.nan
        if k % 2 == 0:
            f[_window_edges(s["times"])[0]] = np.nan
    a = _piece(31, 4, 2400, 1, cuts=([3, 4, 1000], [1000]), edit=nans)
    b = _piece(32, 3, 2400, 101, cuts=([700],))
    c = _piece(33, 2, 2400, 201, t0=T0 + 600 * SEC, cuts=([1000],))
    for pieces in ([a, b], [a, b, c]):
        sd = _desc(pieces)
        lo, hi = _span(pieces)
        for q in [(60 * SEC, 0, lo, hi), (7 * SEC, 0, lo, hi), (0, 0, lo, hi)]:
            for calls in [[(f, F)] for f in ALL6] + [[("min", F), ("max", F)], [("sum", F), ("max", F), ("first", F), ("count", I)]]:
                got = _merged(pieces, calls, q, f"nan x{len(pieces)} {calls} iv={q[0]}", sd=sd)
                if calls == [("sum", F)]:
                    assert np.isnan(np.asarray(got["cols"][0]["values"]).view(np.float64)).any(), "NaN reached the merged sums"
    a.close(); b.close(); c.close()


def test_integer_sums_that_wrap_int64_across_shards():
    """A <- B where each shard's sum fits int64 and the total does not: 2 series x 1000 rows of ~4.15e15 (~0.9 * 2^63 per shard),
    then the same below zero.  Go's int64 sum wraps; the oracle restates it.  The oracle scans [A, B]."""
    for sign in (1, -1):
        def big(k, s):
            s["cols"][I] = (sign * (4_150_000_000_000_000 + np.random.default_rng(k).integers(-1000, 1000, s["times"].size)).astype(np.int64),
                            s["cols"][I][1])
        a = _piece(41, 2, 1000, 1, edit=big)
        b = _piece(42, 2, 1000, 101, edit=lambda k, s: big(k + 7, s))
        sd = _desc([a, b])
        lo, hi = _span([a, b])
        exact = [sum(int(x) for s in p.series for x in s["cols"][I][0]) for p in (a, b)]
        assert all(-2**63 <= e < 2**63 for e in exact) and not -2**63 <= sum(exact) < 2**63, exact
        for q in [(0, 0, lo, hi), (600 * SEC, 0, lo, hi)]:
            for calls in ([("sum", I)], [("sum", I), ("count", I), ("sum", F)]):
                got = _merged([a, b], calls, q, f"wrap {sign} {calls} iv={q[0]}", sd=sd)
                if q[0] == 0:
                    assert int(np.asarray(got["cols"][0]["values"]).view(np.int64)[0]) == (sum(exact) + 2**63) % 2**64 - 2**63
        a.close(); b.close()


@pytest.mark.parametrize("direction", ["merged-in", "merged-into"])
def test_a_shard_without_rows_in_range(direction):
    """E has rows, but none in the query range.  merged-in: A <- E; merged-into: E <- A.  Either way the result is A's own record
    bitwise -- single-call selectors keep A's row times, not the window starts E's empty record holds.  The oracle scans [A, E]
    or [E, A]; float sums: E + A or A + E, i.e. A's"""
    a = _piece(51, 4, 2400, 1, nulls=NULLS, cuts=([1000], [333, 1000]))
    e = _piece(52, 3, 2400, 101, t0=T0 + 100_000 * SEC)
    pieces = [a, e] if direction == "merged-in" else [e, a]
    sd = _desc(pieces)
    lo, hi = _span([a])
    for q in [(60 * SEC, 0, lo, hi), (0, 0, lo, hi), (60 * SEC, 13 * SEC, lo + 611 * SEC, hi - 397 * SEC)]:
        for calls in SINGLE + MIXED:
            got = _merged(pieces, calls, q, f"empty {direction} {calls} iv={q[0]}", sd=sd)
            own = _query(a, calls, q[0], q[2], q[3], q[1])
            _same(got, own.dense_host(), f"empty {direction} {calls} iv={q[0]}: A's record")
            own.close()
    a.close(); e.close()


def test_a_field_that_one_shard_never_wrote():
    """A <- B where B has no F pages (page_len 0 in every segment), and B' <- A where B' has no I pages.  The oracle scans
    [A, B] / [B', A]; float sums: B + A (B adds nothing) and A + B'"""
    a = _piece(61, 4, 2400, 1, nulls=NULLS, cuts=([1000], [333, 1000]))
    b = _piece(62, 3, 2400, 101, t0=T0 + 300 * SEC, cuts=([700],), absent=[F])
    b2 = _piece(63, 3, 2400, 201, t0=T0 + 300 * SEC, cuts=([1000, 31],), absent=[I])
    for pieces in ([a, b], [b2, a]):
        sd = _desc(pieces)
        lo, hi = _span(pieces)
        for q in [(60 * SEC, 0, lo, hi), (0, 0, lo, hi)]:
            for calls in SINGLE + MIXED:
                _merged(pieces, calls, q, f"absent {[p.absent for p in pieces]} {calls} iv={q[0]}", sd=sd)
    a.close(); b.close(); b2.close()


@pytest.mark.parametrize("mapped", [False, True], ids=["one-tagset", "map"])
def test_chain_of_three_shards(mapped):
    """A <- B <- C: A and B over one range, C starting 1100 s later; under the map A's series go to [0, 1, 2, 0, 1], B's to
    [2, 2, 0, 0], C's to [1, 0, 1].  The oracle scans [A, B, C]; float sums: C + (B + A)"""
    a, b = _pair(False, NULLS, mapped=mapped)
    c = _piece(3, 3, 2400, 201, t0=T0 + 1100 * SEC, nulls=NULLS, cuts=([1000], [4, 1000]), groups=[1, 0, 1] if mapped else None)
    sd = _desc([a, b, c])
    for q in _grid_queries(*_span([a, b, c])):
        for calls in MIXED + SINGLE:
            _merged([a, b, c], calls, q, f"chain {calls} iv={q[0]} off={q[1]}", mapped=mapped, sd=sd)
    a.close(); b.close(); c.close()


@pytest.mark.parametrize("ascending", [True, False], ids=["asc", "desc"])
def test_records_after_a_merge(ascending):
    """A <- B under the map; og_query_next runs once before the merge (the host copy of A's record is filled), then the records
    are read again at chunk_size 7: they are the merged record's cells, latest window first when descending.  The merged
    record itself is checked as everywhere: the oracle scans [A, B]; float sums: B + A"""
    a, b = _pair(True, NULLS, mapped=True)
    sd = _desc([a, b])
    lo, hi = _span([a, b])
    for q in [(60 * SEC, 0, lo, hi), (0, 0, lo, hi)]:
        for calls in [MIXED8, [("first", F)], [("max", I)], [("min", B), ("max", I)], [("last", I), ("first", B)]]:
            label = f"records {calls} iv={q[0]} asc={ascending}"
            qa = _query(a, calls, q[0], q[2], q[3], mapped=True, ascending=ascending, chunk_size=7)
            qb = _query(b, calls, q[0], q[2], q[3], mapped=True, ascending=ascending, chunk_size=7)
            next(qa.records())
            _merge(qa, qb)
            got = qa.dense_host()
            _check(got, [a, b], [qa.desc, qb.desc], calls, q, label, True, sd)
            assert_records(list(qa.records()), records_of(got, calls, ascending, 7), label)
            qa.close(); qb.close()
    a.close(); b.close()


def _without_times(dv, c):
    """dv with column c's times removed (a record whose selector carries no time)"""
    cols = (L.DenseCol * dv.n_cols)()
    for k in range(dv.n_cols):
        cols[k] = dv.cols[k]
    cols[c].times = None
    out = L.DenseView(dv.n_groups, dv.n_buckets, dv.start, dv.interval, dv.n_cols, cols, dv.stream)
    out._keep = cols
    return out


def test_merge_refuses_records_of_other_calls_and_leaves_the_record_alone():
    a, b = _pair(False, NULLS)
    lo, hi = _span([a, b])

    def refused(calls_a, calls_b, status, text=None, strip_times=None, b_shift=0):
        qa = _query(a, calls_a, 60 * SEC, lo, hi)
        qb = _query(b, calls_b, 60 * SEC, lo + b_shift, hi + b_shift)
        before = qa.dense_host()
        dv = qb.dense_view() if strip_times is None else _without_times(qb.dense_view(), strip_times)
        assert L.lib().og_query_merge_dense(qa.h, C.byref(dv)) == status, (calls_a, calls_b)
        if text:
            assert text in L.lib().og_last_error().decode(), (calls_a, calls_b, L.lib().og_last_error())
        _same(qa.dense_host(), before, f"refused {calls_a} <- {calls_b}")
        qa.close(); qb.close()

    refused([("sum", F), ("sum", I)], [("sum", F), ("count", I)], L.OG_E_INVAL, "dense column 1")   # a count into a sum
    refused([("first", F)], [("last", F)], L.OG_E_INVAL, "dense column 0")                         # a first into a last
    refused([("min", F)], [("min", I)], L.OG_E_INVAL, "dense column 0")                            # int bits as doubles
    refused([("count", F), ("max", I), ("sum", F)], [("count", F), ("max", B), ("sum", F)], L.OG_E_INVAL, "dense column 1")
    refused([("sum", F)], [("sum", F), ("count", F)], L.OG_E_INVAL)                                # another n_calls
    refused([("first", F), ("count", I)], [("first", F), ("count", I)], L.OG_E_INVAL, "times", strip_times=0)
    refused([("max", F)], [("max", F)], L.OG_E_INVAL, "grids differ", b_shift=60 * SEC)             # same shape, another start
    # before og_query_run there is no record to merge into
    qa = _query(a, [("max", F)], 60 * SEC, lo, hi, run=False)
    qb = _query(b, [("max", F)], 60 * SEC, lo, hi)
    before_b = qb.dense_host()
    assert L.lib().og_query_merge_dense(qa.h, C.byref(qb.dense_view())) == L.OG_E_STATE
    _same(qb.dense_host(), before_b, "merge before run: the other record")
    own = _query(a, [("max", F)], 60 * SEC, lo, hi)
    _same(qa.run().dense_host(), own.dense_host(), "merge before run, then run")
    qa.close(); qb.close(); own.close()
    # counts of columns of different types are both OG_AGG_COUNT / OG_TYPE_INT: they merge, adding the counts
    qa, qb = _query(a, [("count", F)], 60 * SEC, lo, hi), _query(b, [("count", B)], 60 * SEC, lo, hi)
    ra, rb = oracle.scan(a.sd, qa.desc, threads=1)["cols"][0], oracle.scan(b.sd, qb.desc, threads=1)["cols"][0]
    _merge(qa, qb)
    got = qa.dense_host()["cols"][0]
    ok = (ra["valid"] != 0) | (rb["valid"] != 0)
    assert np.array_equal(got["valid"] != 0, ok)
    assert np.array_equal(got["values"].view(np.int64)[ok], (ra["values"].view(np.int64) * (ra["valid"] != 0) + rb["values"].view(np.int64) * (rb["valid"] != 0))[ok])
    qa.close(); qb.close()
    a.close(); b.close()


# ---------------------------------------------------------------------------------------------------------------
# og_query_allreduce
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("graph", [True, False], ids=["graph", "no-graph"])
def test_allreduce_world1_keeps_the_record(graph, monkeypatch):
    """At world 1 the all-reduce hands back the record it started from, bitwise, selector times included.  Sequence: run ->
    allreduce (the graph is captured) -> merge B in -> allreduce (replayed: it must see the merged record) -> run -> allreduce
    (it must see the new run's record, not the merged one)."""
    if not graph:
        monkeypatch.setenv("OGPU_NO_MERGE_GRAPH", "1")
    a, b = _pair(True, NULLS, mapped=True)
    lo, hi = _span([a, b])
    comm = Comm.init_rank(Comm.unique_id(), 0, 1)
    try:
        for calls in [MIXED8, [("first", F)], [("min", B)], [("last", I), ("max", F), ("sum", I)]]:
            label = f"world 1 {calls} graph={graph}"
            q = _query(a, calls, 60 * SEC, lo, hi, mapped=True)
            qb = _query(b, calls, 60 * SEC, lo, hi, mapped=True)
            own = q.dense_host()
            comm.allreduce(q)
            _same(q.dense_host(), own, label + " first allreduce")
            _merge(q, qb)
            merged = q.dense_host()
            _check(merged, [a, b], [q.desc, qb.desc], calls, (60 * SEC, 0, lo, hi), label, True)
            comm.allreduce(q)
            _same(q.dense_host(), merged, label + " after the merge")
            q.run()
            comm.allreduce(q)
            _same(q.dense_host(), own, label + " after a new run")
            q.close(); qb.close()
    finally:
        comm.close()
    a.close(); b.close()


W2_CALLS = [MIXED8, [("first", F)], [("min", I), ("max", B)], [("sum", I), ("last", F)]]
W2_ROWS = 2400


def _w2_piece(rank):
    """rank r's shard: A (rank 0) or B (rank 1) of the mapped, shifted pair, nulls in every column"""
    if rank == 0:
        return _piece(1, 5, W2_ROWS, 1, nulls=NULLS, cuts=([1000], [333, 1000]), groups=[0, 1, 2, 0, 1])
    return _piece(2, 4, W2_ROWS, 101, t0=T0 + 1700 * SEC, nulls=NULLS, cuts=([700], [1000, 31]), groups=[2, 2, 0, 0])


W2_RANGE = (T0, T0 + 1700 * SEC + (W2_ROWS - 1) * SEC)


def _rank_main(rank, world, idfile, out):
    import time
    Shard.init(rank)
    if rank == 0:
        uid = Comm.unique_id()
        with open(idfile + ".tmp", "wb") as f:
            f.write(uid)
        os.replace(idfile + ".tmp", idfile)
    else:
        for _ in range(600):
            if os.path.exists(idfile):
                break
            time.sleep(0.05)
        uid = open(idfile, "rb").read()
    comm = Comm.init_rank(uid, rank, world)
    p = _w2_piece(rank)
    res = []
    for calls in W2_CALLS:
        q = _query(p, calls, 60 * SEC, *W2_RANGE, mapped=True)
        comm.allreduce(q)
        d = q.dense_host()
        res.append(dict(n_groups=d["n_groups"], n_buckets=d["n_buckets"], start=d["start"],
                        cols=[dict(values=c["values"].view(np.uint64).copy(), valid=c["valid"].copy(),
                                   times=None if c["times"] is None else c["times"].copy()) for c in d["cols"]]))
        q.close()
    comm.close(); p.close()
    out.put((rank, res))


def test_allreduce_two_gpus_mixed_types_and_tagset_map():
    """Two ranks, one shard each: A on rank 0, B on rank 1 (mapped, shifted, nulls).  Each rank's record must be what the oracle's
    scan of [A, B] gives; float sums: B + A (two partial sums added once: either order gives these bits); every rank the same bits."""
    if L.lib().og_device_count() < 2:
        pytest.skip("needs two GPUs")
    import multiprocessing as mp
    ctx = mp.get_context("spawn")
    out = ctx.Queue()
    world = 2
    with tempfile.TemporaryDirectory() as td:
        idfile = os.path.join(td, "nccl_id")
        procs = [ctx.Process(target=_rank_main, args=(r, world, idfile, out)) for r in range(world)]
        for p in procs:
            p.start()
        try:
            got = dict(out.get(timeout=300) for _ in range(world))
        finally:
            for p in procs:
                p.join(timeout=60)
                if p.is_alive():
                    p.terminate()
                    p.join(timeout=10)
        assert all(p.exitcode == 0 for p in procs), [p.exitcode for p in procs]
    pieces = [_w2_piece(0), _w2_piece(1)]
    sd = _desc(pieces)
    for ci, calls in enumerate(W2_CALLS):
        qs = [_query(p, calls, 60 * SEC, *W2_RANGE, mapped=True, run=False) for p in pieces]
        for r in range(world):
            _check(got[r][ci], pieces, [x.desc for x in qs], calls, (60 * SEC, 0) + W2_RANGE, f"world 2 rank {r} {calls}", True, sd)
        _same(got[1][ci], got[0][ci], f"world 2 {calls}: ranks agree")
        for x in qs:
            x.close()
    for p in pieces:
        p.close()
