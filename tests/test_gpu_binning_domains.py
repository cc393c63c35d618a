"""Every aggregate path on shards of more than 4096 series, against the oracle: several binning domains, chunk plans, block merges.

The interleaved copy of a float column bins segments by domain: segment index j of a block of OG_IL_SUPER = 4096 consecutive
series when every series has J segments, the whole shard otherwise.  configs[1] (5000 series) holds two such blocks, and code
only reached above 4096 series is checked here: the domain index and per-domain time alignment of k_il_scan, the folded column of
a lane group (k_il_assign), the lane groups each chunk launches, the folded matrix with several blocks, chunk sizes rounded to
4096 or to 32, the block merge that switches on above 512 series, and the general-segment list cut per chunk.

Shards: 100-row segments at a 1 s cadence (segments of <= 1024 rows keep two-column queries on k_fused_cols), five columns:
  c0 FLOAT G-hi (packed lanes), c1 FLOAT G-lo (Gorilla lanes), c2 FLOAT G-hi with 1 permille nulls (about 10 % of the segments
  have a null and are general segments in every domain), c3 INT walk, c4 BOOL.
Shards of several pieces (another time grid for one block, one series off the grid, ragged series) concatenate the arrays of
several HostShards; the oracle reads the same arrays.

Each query asserts the path it means to take from og_stats, then compares the dense record with oracle.scan(threads=1):
bitwise under OG_Q_STRICT_ORDER, and in every order of one tagset that is not the reference's (the folded order of path 3, the
block merge of the other paths) float sums within test_gpu_parity's SUM_RTOL.  Every oracle answer is computed once per shard and
query and reused across chunk plans."""
import os
from concurrent.futures import ThreadPoolExecutor
from typing import NamedTuple

import numpy as np
import pytest

import oracle
from opengemini_b200 import AggQuery, Shard
from opengemini_b200 import _lib as L
from test_gpu_packed_lanes import _form, _model
from test_gpu_parity import compare_dense

pytestmark = pytest.mark.gpu

T0, SEC = 1_700_000_000_000_000_000, 1_000_000_000
SUPER, ROWS = 4096, 100  # OG_IL_SUPER; rows per segment
ALL6 = ("count", "sum", "min", "max", "first", "last")
BOOL_FUNCS = ("count", "min", "max", "first", "last")
COLS = [(L.TYPE_FLOAT, L.SYNTH_F_HI, 0), (L.TYPE_FLOAT, L.SYNTH_F_LO, 0), (L.TYPE_FLOAT, L.SYNTH_F_HI, 1),
        (L.TYPE_INT, L.SYNTH_INT_WALK, 0), (L.TYPE_BOOL, L.SYNTH_BOOL, 0)]
THREADS = max(1, min(16, len(os.sched_getaffinity(0))))

# id: pieces of (series, segments per series, time shift in ns), folded (the default one-tagset query takes path 3)
SHARDS = {
    "A_4095": ([(4095, 1, 0)], True),                                 # one domain, last lane group of 31 lanes
    "B_4096": ([(4096, 2, 0)], True),                                 # exactly one full block
    "C_4097": ([(4097, 2, 0)], True),                                 # a second block of one series
    "D_4129": ([(4129, 3, 0)], True),                                 # a second block of one full group and one lane
    "E_8292": ([(8292, 3, 0)], True),                                 # three blocks, general segments (c2) in all of them
    "F_shifted_block": ([(4096, 3, 0), (700, 3, 37_250_000_000)], True),  # each block on its own grid: still folded
    "G_one_series_off": ([(4096, 3, 0), (699, 3, 0), (1, 3, SEC // 2)], False),  # not aligned: path 2, block merge
    "H_ragged": ([(4000, 3, 0), (300, 2, 0)], False),                 # J == 0: one domain over the whole shard
}


@pytest.fixture(scope="module", autouse=True)
def _device():
    Shard.init(0)


# ---------------------------------------------------------------------------------------------------------------
# shards
# ---------------------------------------------------------------------------------------------------------------
def _host_export(hs):
    """the arrays of a HostShard in the layout of Shard.export()"""
    d = hs.desc
    ns, ng, nc = d.n_series, d.n_segments, d.n_columns

    def arr(p, n):
        return np.ctypeslib.as_array(p, shape=(n,)).copy()
    return dict(data=arr(d.data, d.data_len), sids=arr(d.sids, ns), series_seg_begin=arr(d.series_seg_begin, ns + 1),
                seg_tmin=arr(d.seg_tmin, ng), seg_tmax=arr(d.seg_tmax, ng),
                page_off=np.stack([arr(d.columns[c].page_off, ng) for c in range(nc)] + [arr(d.time_page_off, ng)]),
                page_len=np.stack([arr(d.columns[c].page_len, ng) for c in range(nc)] + [arr(d.time_page_len, ng)]),
                col_types=np.array([d.columns[c].type for c in range(nc)], np.int32))


def _concat(exs):
    """one shard of the pieces' series in order: sids, segment indices and page offsets shifted past the earlier pieces"""
    data_base = np.cumsum([0] + [e["data"].size for e in exs[:-1]]).astype(np.uint64)
    sid_base = np.cumsum([0] + [e["sids"].size for e in exs[:-1]]).astype(np.uint64)
    seg_base = np.cumsum([0] + [e["seg_tmin"].size for e in exs[:-1]]).astype(np.uint32)
    return dict(data=np.concatenate([e["data"] for e in exs]), sids=np.concatenate([e["sids"] + k for e, k in zip(exs, sid_base)]),
                series_seg_begin=np.concatenate([exs[0]["series_seg_begin"][:1]] +
                                                [e["series_seg_begin"][1:] + k for e, k in zip(exs, seg_base)]).astype(np.uint32),
                seg_tmin=np.concatenate([e["seg_tmin"] for e in exs]), seg_tmax=np.concatenate([e["seg_tmax"] for e in exs]),
                page_off=np.concatenate([e["page_off"] + k for e, k in zip(exs, data_base)], axis=1),
                page_len=np.concatenate([e["page_len"] for e in exs], axis=1), col_types=exs[0]["col_types"])


class Case:
    def __init__(self, name):
        pieces, self.folds = SHARDS[name]
        seed = 1 + sum(map(ord, name))
        hss = [oracle.HostShard(n, j * ROWS, COLS, t0=T0 + shift, dt=SEC, seed=seed + 7 * i, rows_per_segment=ROWS, threads=THREADS)
               for i, (n, j, shift) in enumerate(pieces)]
        if len(hss) == 1:
            self.sh, self.sd, ex = Shard.open_desc(hss[0].desc, keepalive=hss[0]), hss[0].desc, _host_export(hss[0])
        else:
            ex = _concat([_host_export(h) for h in hss])
            nc = len(COLS)
            self.sh = Shard.open(ex["data"], ex["sids"], ex["series_seg_begin"], ex["seg_tmin"], ex["seg_tmax"],
                                 [(f"c{c}", int(ex["col_types"][c]), ex["page_off"][c], ex["page_len"][c]) for c in range(nc)],
                                 ex["page_off"][nc], ex["page_len"][nc])
            self.sd = oracle.shard_desc_from_export(ex)
        self.ex, self._hosts = ex, hss  # a HostShard owns the arrays its desc points at
        self.n = ex["sids"].size
        ssb = ex["series_seg_begin"]
        per = np.diff(ssb)
        self.J = int(per[0]) if np.all(per == per[0]) else 0
        self.lo, self.hi = T0, int(ex["seg_tmax"].max())
        self.groups = {"mod7": (np.arange(self.n) % 7, 7), "block": (np.arange(self.n) // SUPER, (self.n + SUPER - 1) // SUPER)}
        self.refs = {}
        self._pages = {}

    def pages(self, col):
        """pages[series][segment] of a column"""
        if col not in self._pages:
            e, ssb = self.ex, self.ex["series_seg_begin"]
            off, ln = e["page_off"][col], e["page_len"][col]
            self._pages[col] = [[e["data"][int(off[g]):int(off[g]) + int(ln[g])] for g in range(ssb[s], ssb[s + 1])] for s in range(self.n)]
        return self._pages[col]

    def general(self, col):
        """(series, segment index) of the pages the interleaved copy does not take"""
        key = ("general", col)
        if key not in self._pages:
            self._pages[key] = [(s, j) for s, segs in enumerate(self.pages(col)) for j, p in enumerate(segs) if _form(p)[0] is None]
        return self._pages[key]

    def domain(self, s, j):
        return (s // SUPER) * self.J + j if self.J else 0


_CASES = {}


@pytest.fixture(scope="module")
def cases():
    yield _CASES
    for c in _CASES.values():
        c.sh.close()
    _CASES.clear()


@pytest.fixture(params=list(SHARDS))
def case(request, cases):
    name = request.param
    if name not in cases:
        cases[name] = Case(name)
    return cases[name]


# ---------------------------------------------------------------------------------------------------------------
# queries
# ---------------------------------------------------------------------------------------------------------------
class Q(NamedTuple):
    """one query: calls ((func, column), ...), interval in seconds, range (None: the shard's), offset in ns, group mode
    ('all', 'series', or a key of Case.groups), filter (RPN tuple or None)"""
    calls: tuple
    iv: int
    rng: tuple = None
    offset: int = 0
    group: str = "all"
    flt: tuple = None


def _q(funcs, col, iv, **kw):
    return Q(tuple((f, col) for f in funcs), iv, **kw)


def _kw(case, q):
    lo, hi = q.rng or (case.lo, case.hi)
    kw = dict(calls=list(q.calls), interval=q.iv * SEC, tmin=lo, tmax=hi, offset=q.offset, filter=list(q.flt) if q.flt else None)
    if q.group in case.groups:
        sg, ng = case.groups[q.group]
        kw.update(group="map", series_group=sg, n_groups=ng)
    else:
        kw.update(group=q.group)
    return kw


def _refs(case, qs):
    """oracle answers of the queries not answered yet, on the host's threads at once (the oracle's ctypes calls let go of the GIL)"""
    todo = [q for q in dict.fromkeys(qs) if q not in case.refs]
    if not todo:
        return
    handles = [AggQuery(case.sh, **_kw(case, q)) for q in todo]
    try:
        with ThreadPoolExecutor(THREADS) as ex:
            for q, r in zip(todo, ex.map(lambda h: oracle.scan(case.sd, h.desc, threads=1), handles)):
                case.refs[q] = r
    finally:
        for h in handles:
            h.close()


def _run(case, q, flags, path, monkeypatch, label, reruns=0):
    """run q the way `path` names (path 4: OGPU_NO_COLS), assert the path and the interleaved copy's counts, compare with the
    oracle; reruns: run the same plan again (scratch reuse).  Returns og_stats."""
    _refs(case, [q])
    ref = case.refs[q]
    col = q.calls[0][1]
    strict = bool(flags & L.Q_STRICT_ORDER)
    exact = strict or q.group != "all"  # one tagset without the strict order: folded (path 3) or block merge (> 512 series)
    with monkeypatch.context() as m:
        if path == 4:
            m.setenv("OGPU_NO_COLS", "1")
        h = AggQuery(case.sh, **_kw(case, q), flags=flags)
        try:
            for k in range(1 + reruns):
                h.run()
                st = h.stats()
                lab = f"{label} {q} flags={flags} run {k}"
                assert st["path"] == path, f"{lab}: path {st['path']}, wanted {path}"
                if path in (2, 3):
                    assert st["il_state"] == 1, lab
                    assert st["general_segments"] == len(case.general(col)), f"{lab}: {st['general_segments']} general segments"
                if path == 3 and q.iv in (60, 1000, 0) and not case.general(col):  # general segments write per-series cells
                    assert st["per_series_cells_used"] == 0, lab
                if path == 3 and q.iv == 3:  # 34 windows a segment, more than OG_IL_WCAP: those lanes leave the fold
                    assert st["per_series_cells_used"] == 1, lab
                compare_dense(h.dense_host(), ref, q.calls, len(q.calls) > 1, f"{lab} [path {path}]", float_sum_exact=exact)
        finally:
            h.close()
    return st


CALLSETS = [(f,) for f in ALL6] + [("sum", "count", "max"), ("sum", "count", "min", "max"), ALL6, ("max", "count")]
IVS = (60, 7, 3, 1000, 0)


def _il_queries(col):
    return [_q(fs, col, iv) for iv in IVS for fs in CALLSETS]


# ---------------------------------------------------------------------------------------------------------------
# the interleaved copy
# ---------------------------------------------------------------------------------------------------------------
def test_interleaved_copy_matches_the_model(case, monkeypatch):
    """il_packed_segments and il_bytes equal _model(), which bins by 4096-series domains; the general segments are the pages
    _form() finds not eligible: none in c0 and c1, about 10 % of c2's, spread over every domain"""
    nseg = case.ex["seg_tmin"].size
    for col in (0, 1, 2):
        q = _q(("count",), col, 0)
        st = _run(case, q, 0, 3 if case.folds else 2, monkeypatch, f"copy c{col}")
        model = _model(case.pages(col))
        assert (st["il_packed_segments"], st["il_bytes"]) == model, f"c{col}: {st['il_packed_segments']}, {st['il_bytes']} != {model}"
        gen = case.general(col)
        if col in (0, 1):
            assert not gen
        else:
            assert 0.05 * nseg < len(gen) < 0.15 * nseg, len(gen)
            doms = {case.domain(s, j) for s, j in gen}
            n_dom = ((case.n + SUPER - 1) // SUPER) * case.J if case.J else 1
            assert len(doms) > 1 or n_dom == 1, f"general segments in {len(doms)} of {n_dom} domains"
            if case.n > 2 * SUPER:
                assert len(doms) == n_dom, f"general segments in {len(doms)} of {n_dom} domains"
        if col == 0:
            assert model[0] == nseg  # G-hi: every segment is packed
        if col == 1:
            assert model[0] < nseg  # G-lo: Gorilla lanes


# ---------------------------------------------------------------------------------------------------------------
# k_fused_il: path 3 (folded) and path 2 (strict order; the default where the shard does not fold)
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("col", [0, 1, 2])
def test_fused_il_every_call_set_and_interval(case, col, monkeypatch):
    """every launch_fast instance (count; sum,count; sum,count,max; sum,count,min,max; max,count and min,count with times; all
    six) at windows inside a segment, 15 and 34 a segment, over every segment, and none; folded queries run twice"""
    qs = _il_queries(col)
    _refs(case, qs)
    for q in qs:
        _run(case, q, L.Q_STRICT_ORDER, 2, monkeypatch, f"c{col}")
        _run(case, q, 0, 3 if case.folds else 2, monkeypatch, f"c{col}", reruns=1 if case.folds else 0)


def test_offset_and_a_range_cut_inside_segments(case, monkeypatch):
    """GROUP BY time(1m, 7s) over a range that starts and ends inside a segment"""
    lo, hi = case.lo + 17 * SEC + SEC // 2, case.hi - 23 * SEC - 1
    qs = [_q(fs, col, 60, rng=(lo, hi), offset=7 * SEC) for col in (0, 1, 2) for fs in (ALL6, ("sum", "count", "max"), ("first",))]
    _refs(case, qs)
    for q in qs:
        _run(case, q, L.Q_STRICT_ORDER, 2, monkeypatch, "cut range")
        _run(case, q, 0, 3 if case.folds else 2, monkeypatch, "cut range", reruns=1 if case.folds else 0)


# ---------------------------------------------------------------------------------------------------------------
# the general paths, the multi-column paths, tag groups and per-series output
# ---------------------------------------------------------------------------------------------------------------
def _general_queries():
    out = []
    for col in (2, 3):
        out += [_q(ALL6, col, iv) for iv in (60, 7, 0)] + [_q(fs, col, 60) for fs in (("sum", "count", "max"), ("min",), ("last",))]
    return out


def test_pull_iterator_and_tile_paths_with_the_block_merge(case, monkeypatch):
    """path 1 (OG_Q_NO_FAST) and path 0 (OG_Q_NO_FUSED), one tagset, order not pinned: above 512 series the per-series cells are
    folded by blocks of 256 series and the block partials by k_merge_folded"""
    qs = _general_queries()
    _refs(case, qs)
    for q in qs:
        _run(case, q, L.Q_NO_FAST, 1, monkeypatch, "path 1")
        _run(case, q, L.Q_NO_FUSED, 0, monkeypatch, "path 0")


WHERE_C0 = (("term", 0, ">", 100.5),)
WHERE_C3_C4 = (("term", 3, ">", 0), ("term", 4, "=", 1), "or")


def _multi_queries():
    two = (("sum", 0), ("count", 0), ("max", 3), ("first", 3))
    sel = (("min", 0), ("last", 0), ("sum", 3), ("count", 3))
    bools = (("sum", 3), ("count", 4), ("min", 4), ("max", 4), ("first", 4), ("last", 4))
    return ([(Q(two, iv, flt=WHERE_C0), 5) for iv in (60, 3, 0)] + [(Q(sel, 1000, flt=WHERE_C0), 5)] +
            [(Q(two, iv, flt=WHERE_C0), 4) for iv in (60, 0)] + [(Q(bools, iv, flt=WHERE_C3_C4), 4) for iv in (60, 7)] +
            [(Q(tuple((f, 4) for f in BOOL_FUNCS), 60, flt=WHERE_C3_C4), 4)])


def test_column_at_a_time_and_multi_column_kernels(case, monkeypatch):
    """path 5: c0 and c3 with WHERE c0 > 100.5; path 4: the same under OGPU_NO_COLS, and c3 with the bool c4 under two terms"""
    qs = _multi_queries()
    _refs(case, [q for q, _ in qs])
    for q, path in qs:
        _run(case, q, L.Q_STRICT_ORDER, path, monkeypatch, "multi")
        _run(case, q, 0, path, monkeypatch, "multi")


def _group_queries():
    """(query, path): k_fused_il serves the float columns without folding (path 2), the pull-iterator kernel the int column"""
    return [(_q(ALL6, 0, 60, group="series"), 2), (_q(("sum", "count", "last"), 2, 7, group="series"), 2),
            (_q(("sum", "count", "max"), 0, 60, group="mod7"), 2), (_q(("min", "first"), 2, 3, group="mod7"), 2),
            (_q(ALL6, 0, 7, group="block"), 2), (_q(("sum", "count", "max"), 3, 60, group="block"), 1)]


def _check_records(case, q, label):
    """per-series output drained through og_query_next once: each record's sid is its series', and its cells are the dense ones"""
    h = AggQuery(case.sh, **_kw(case, q)).run()
    try:
        d = h.dense_host()
        nb = d["n_buckets"]
        seen = np.zeros(case.n, bool)
        for rec in h.records():
            g = rec["group"]
            assert rec["sid"] == int(case.ex["sids"][g]), f"{label}: record of series {g} carries sid {rec['sid']}"
            seen[g] = True
            cells = g * nb + (rec["times"] - d["start"]) // d["interval"]
            for k in range(len(q.calls)):
                col = rec["cols"][k]
                assert np.array_equal(col["valid"], d["cols"][k]["valid"][cells].astype(bool)), label
                want = d["cols"][k]["values"][cells][col["valid"]]
                assert np.array_equal(col["values"].view(np.uint64), want.view(np.uint64)), label
        any_valid = np.zeros(case.n * nb, bool)
        for c in d["cols"]:
            any_valid |= c["valid"].astype(bool)
        assert np.array_equal(seen, any_valid.reshape(case.n, nb).any(1)), label
    finally:
        h.close()


def test_group_modes(case, monkeypatch):
    """per-series output (up to 8292 tagsets), tag groups of series % 7, and one tag group per block of 4096 series"""
    qs = _group_queries()
    _refs(case, [q for q, _ in qs])
    for q, path in qs:
        _run(case, q, L.Q_STRICT_ORDER, path, monkeypatch, "groups")
        _run(case, q, 0, path, monkeypatch, "groups")
    _check_records(case, qs[0][0], "records")


# ---------------------------------------------------------------------------------------------------------------
# chunk plans
# ---------------------------------------------------------------------------------------------------------------
def _chunk_queries(case):
    default = 3 if case.folds else 2
    return ([(_q(("sum", "count", "max"), 0, 60), 0, default), (_q(("sum", "count", "max"), 0, 60), L.Q_STRICT_ORDER, 2)] +
            [(_q(("last",), 2, iv), 0, default) for iv in (3, 1000)] + [(_q(ALL6, 1, iv), 0, default) for iv in (3, 1000)] +
            [(_q(ALL6, 2, 60), L.Q_NO_FAST, 1), (_q(("sum", "count", "max"), 3, 60), L.Q_NO_FUSED, 0)] +
            [(q, 0, path) for i, (q, path) in enumerate(_multi_queries()) if i in (0, 4, 6)] +
            [(q, 0, path) for q, path in _group_queries()[::2]])


@pytest.mark.parametrize("chunk", ["4096", "5000", "1000", "33"])
def test_chunk_plans(case, chunk, monkeypatch):
    """OGPU_CHUNK_SERIES: 4096 and 5000 (rounded down to 4096) give chunks of whole blocks; 1000 (rounded to 992) and 33 (32) cut
    blocks, so lane groups, sorted by stream length, straddle chunks and run once per chunk with the lanes of each"""
    monkeypatch.setenv("OGPU_CHUNK_SERIES", chunk)
    qs = _chunk_queries(case)
    _refs(case, [q for q, _f, _p in qs])
    for q, flags, path in qs:
        _run(case, q, flags, path, monkeypatch, f"chunks of {chunk}", reruns=1 if path == 3 else 0)
