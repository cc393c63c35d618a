"""Tagset queries (GROUP BY <tag>: OG_GROUP_MAP, and per-series output, OG_GROUP_PER_SERIES) against the oracle, on maps of every
shape, every aggregate path, chunk plans that cut tagsets, and the records og_query_next slices them into.

A tagset query folds each tagset's series in shard order (k_merge_groups, k_merge_per_series), the reference's cross-series order
(reccord_functions.go), whatever the flags.  So every dense record here is compared with oracle.scan bit for bit, float sums
included, and og_stats' rows_decoded and page_bytes with the oracle's.  Every query asserts the path it takes.

Maps: the identity (which must equal per-series output bitwise), one tagset (which must equal OG_GROUP_ALL under
OG_Q_STRICT_ORDER bitwise), unused ids at the front, middle and end of the id range, three times as many ids as series, tagsets
of 1, 15, 16, 17, 31, 32, 33 and 257 members around k_merge_groups' 16-load batches (contiguous, and strided over the whole
shard), ids permuted against series order, one big tagset with a few singletons, and 1500 tagsets over 4500 series (two
OG_IL_SUPER blocks of the interleaved copy).

Shards: a regular one (Shard.synth and its oracle.HostShard twin), a ragged one with series of 0 to 6 segments and a run of 64
series without segments, and one without series.  Oracle answers are computed once per shard, map and query, on the host's
threads at once (each scan single-threaded: a multi-threaded scan merges its workers' partials, another float sum order)."""
import ctypes as C
import os
from concurrent.futures import ThreadPoolExecutor
from typing import NamedTuple

import numpy as np
import pytest

import oracle
import segment_shards as ss
from opengemini_b200 import AggQuery, Shard
from opengemini_b200 import _lib as L
from records_model import assert_records, records_of
from test_gpu_parity import compare_dense

pytestmark = pytest.mark.gpu

T0, SEC = ss.T0, ss.SEC
THREADS = max(1, min(16, len(os.sched_getaffinity(0))))
ALL6 = ("count", "sum", "min", "max", "first", "last")
BOOL5 = ("count", "min", "max", "first", "last")
BATCH = (1, 15, 16, 17, 31, 32, 33, 257)  # around k_merge_groups' batches of U = 16 loads

# c0 FLOAT G-hi, c1 FLOAT G-lo with a null in about a third of the segments (general segments beside the interleaved copy),
# c2 INT walk with 3 % nulls, c3 BOOL with 10 % nulls
SYNTH_COLS = [(L.TYPE_FLOAT, L.SYNTH_F_HI, 0), (L.TYPE_FLOAT, L.SYNTH_F_LO, 1), (L.TYPE_INT, L.SYNTH_INT_WALK, 30),
              (L.TYPE_BOOL, L.SYNTH_BOOL, 100)]
RAGGED_KINDS, RAGGED_NULLS = ["f_hi", "f_lo", "i_s8b", "bool"], [0.0, 0.001, 0.03, 0.1]


@pytest.fixture(scope="module", autouse=True)
def _device():
    Shard.init(0)


# ---------------------------------------------------------------------------------------------------------------
# shards
# ---------------------------------------------------------------------------------------------------------------
def _sids(sh):
    n = sh.info()["n_series"]
    sids = np.empty(n, np.uint64)
    L.check(L.lib().og_shard_export(sh.h, None, sids.ctypes.data, None, None, None, None, None, None), "og_shard_export")
    return sids


class Case:
    """an open shard, the host description the oracle scans, and the oracle's answers so far"""

    def __init__(self, name, sh, sd, late, keep):
        self.name, self.sh, self.sd, self.keep = name, sh, sd, keep
        info = sh.info()
        self.n, tmax = info["n_series"], info["tmax"]
        self.sids = _sids(sh)
        # 'cut' starts and ends inside a segment; 'late' starts `late` seconds in, after the last row of the ragged shard's
        # series of one or two segments
        self.ranges = {"full": (T0, tmax, 0), "cut": (T0 + 23 * SEC + SEC // 2, tmax - 17 * SEC - 1, 7 * SEC),
                       "late": (T0 + late * SEC, tmax, 0)}
        self.refs = {}


def _regular(n, rows, rows_per_segment, seed):
    sh = Shard.synth(n, rows, SYNTH_COLS, t0=T0, dt=SEC, seed=seed, rows_per_segment=rows_per_segment)
    hs = oracle.HostShard(n, rows, SYNTH_COLS, t0=T0, dt=SEC, seed=seed, rows_per_segment=rows_per_segment, threads=THREADS)
    return Case(f"regular {n}", sh, hs.desc, rows // 2, hs)


EMPTY_RUN = (64, 128)  # series without segments: two whole chunks of 32 series, one of 96 cut


def _ragged():
    """192 series of 0 to 6 segments of at most 300 rows (the last one shorter), series 64..127 without segments"""
    rng = np.random.default_rng(71)
    series, lengths = [], []
    for s in range(192):
        k = 0 if EMPTY_RUN[0] <= s < EMPTY_RUN[1] else (3, 1, 4, 1, 5, 2, 6, 0, 2)[s % 9]
        rows = 300 * k - 13 * (s % 5) if k else 0
        series.append(ss.series_rows(rng, rows, RAGGED_KINDS, RAGGED_NULLS))
        lengths.append(ss.mixed([300], rows) if rows else [])
    sh, sd = ss.open_shard(series, ss.types_of(RAGGED_KINDS), lengths)
    ex_ssb = np.diff(sh.export()["series_seg_begin"])
    assert (ex_ssb == 0).sum() >= 64 and not ex_ssb[EMPTY_RUN[0]:EMPTY_RUN[1]].any()
    return Case("ragged", sh, sd, 700, sd)


_CASES = {}


@pytest.fixture(scope="module")
def cases():
    yield _CASES
    for c in _CASES.values():
        c.sh.close()
    _CASES.clear()


def _case(cases, name):
    if name not in cases:
        cases[name] = {"regular": lambda: _regular(600, 1200, 400, 5), "big": lambda: _regular(4500, 200, 100, 9),
                       "ragged": _ragged}[name]()
    return cases[name]


# ---------------------------------------------------------------------------------------------------------------
# maps
# ---------------------------------------------------------------------------------------------------------------
def _spread(sizes):
    """tagset ids of sum(sizes) series, each tagset's members strided over the whole range"""
    key = [((k + 0.5) / m, g) for g, m in enumerate(sizes) for k in range(m)]
    return np.array([g for _f, g in sorted(key)], np.uint32)


def tagset_map(shape, n):
    """(series_group, n_groups) of a map shape over n series; (None, 0) for per-series output"""
    rng = np.random.default_rng(n + sum(map(ord, shape)))
    if shape == "series":
        return None, 0
    if shape == "identity":
        return np.arange(n, dtype=np.uint32), n
    if shape == "one":
        return np.zeros(n, np.uint32), 1
    if shape == "empty_edges":  # ids 0-2, 17-22 and 37-39 unused
        used = np.r_[3:17, 23:37]
        sg = used[rng.integers(0, used.size, n)]
        sg[:used.size] = used  # every other id in use
        return sg.astype(np.uint32), 40
    if shape == "sparse":  # three ids a series: most tagsets empty
        return rng.integers(0, 3 * n, n).astype(np.uint32), 3 * n
    if shape in ("batch_contig", "batch_strided"):
        sizes = list(BATCH) + [n - sum(BATCH)]
        assert sizes[-1] > 0
        if shape == "batch_contig":
            return np.repeat(np.arange(len(sizes)), sizes).astype(np.uint32), len(sizes)
        return _spread(sizes), len(sizes)
    if shape == "permuted":  # series s in tagset perm[s % 37]: ids not monotonic in series order, members spread out
        perm = rng.permutation(37)
        return perm[np.arange(n) % 37].astype(np.uint32), 37
    if shape == "big_singletons":  # tagset 3 holds all series but five singletons
        sg = np.full(n, 3, np.uint32)
        sg[[0, 257, n // 2, n - 2, n - 1]] = [0, 1, 2, 4, 5]
        return sg, 6
    if shape == "thousands":
        return rng.integers(0, 1500, n).astype(np.uint32), 1500
    raise KeyError(shape)


def test_map_shapes_are_what_they_claim():
    sg, ng = tagset_map("empty_edges", 600)
    assert set(np.unique(sg)) == set(range(3, 17)) | set(range(23, 37)) and ng == 40
    sg, ng = tagset_map("sparse", 600)
    assert ng == 1800 and np.unique(sg).size < 600
    for shape in ("batch_contig", "batch_strided"):
        sg, ng = tagset_map(shape, 600)
        assert list(np.bincount(sg, minlength=ng)[:len(BATCH)]) == list(BATCH)
        if shape == "batch_strided":  # every block of 32 series holds a member of every tagset of 32 or more
            for g in range(5, len(BATCH) + 1):
                assert all((sg[a:a + 32] == g).any() for a in range(0, 576, 32)), g
        else:
            assert np.all(np.diff(sg.astype(np.int64)) >= 0)
    sg, ng = tagset_map("permuted", 600)
    assert np.any(np.diff(sg[:37].astype(np.int64)) < 0) and np.unique(sg).size == ng
    sg, ng = tagset_map("big_singletons", 600)
    assert np.bincount(sg).tolist() == [1, 1, 1, 595, 1, 1]
    sg, ng = tagset_map("thousands", 4500)
    assert 1300 < np.unique(sg).size < 1500 and ng == 1500


# ---------------------------------------------------------------------------------------------------------------
# queries
# ---------------------------------------------------------------------------------------------------------------
class Q(NamedTuple):
    """calls ((func, column), ...), interval in seconds, range ('full', 'cut' with a 7 s offset, 'late'), WHERE (RPN), flags,
    OGPU_NO_COLS, the path og_stats must report"""
    calls: tuple
    iv: int
    rng: str
    flt: tuple
    flags: int
    no_cols: bool
    path: int


def _q(calls, iv, path, rng="full", flt=None, flags=0, no_cols=False):
    return Q(tuple(calls), iv, rng, flt, flags, no_cols, path)


def _one(funcs, col):
    return tuple((f, col) for f in funcs)


MULTI = [((("sum", 0), ("count", 2), ("max", 1), ("last", 3), ("min", 2), ("first", 1)), 60, "full", (("term", 2, ">", 0),)),
         ((("count", 3), ("sum", 1), ("first", 3), ("sum", 2)), 7, "cut", (("term", 0, ">", 100.5),)),
         ((("min", 0), ("max", 0), ("sum", 2), ("count", 3)), 0, "late", (("term", 3, "=", 1),))]

QUERIES = (
    # path 2: one float column, the interleaved copy built (no tagset query folds: path 3 never serves a map)
    [_q(_one(ALL6, 0), 60, 2), _q(_one(("sum", "count", "max"), 1), 7, 2), _q(_one(("first",), 0), 0, 2),
     _q(_one(("min",), 1), 60, 2, "cut"), _q(_one(("sum",), 1), 7, 2, "late")] +
    # path 1: an int column, bool selectors, a float column under OG_Q_NO_FAST
    [_q(_one(ALL6, 2), 60, 1), _q(_one(("last",), 2), 7, 1, "cut"), _q(_one(ALL6, 1), 0, 1, flags=L.Q_NO_FAST),
     _q(_one(("sum", "count", "min"), 0), 60, 1, "cut", flags=L.Q_NO_FAST), _q(_one(("first",), 3), 60, 1),
     _q(_one(("max",), 3), 7, 1, "late"), _q(_one(BOOL5, 3), 0, 1)] +
    # path 5: several columns with one WHERE term; path 4: the same without the column-at-a-time kernel
    [_q(c, iv, 5, r, flt) for c, iv, r, flt in MULTI] + [_q(c, iv, 4, r, flt, no_cols=True) for c, iv, r, flt in MULTI] +
    # path 0: the materialisation tile
    [_q(_one(ALL6, 1), 60, 0, flags=L.Q_NO_FUSED), _q(_one(BOOL5, 3), 7, 0, "cut", flags=L.Q_NO_FUSED),
     _q((("sum", 2), ("last", 0)), 0, 0, flags=L.Q_NO_FUSED),
     _q((("sum", 0), ("count", 2), ("first", 1)), 60, 0, "late", (("term", 3, "=", 1),), flags=L.Q_NO_FUSED)])
PATH_QUERIES = [QUERIES[i] for i in (0, 5, 12, 15, 18)]  # one query on each path


def _kw(case, shape, q, **extra):
    tmin, tmax, offset = case.ranges[q.rng]
    kw = dict(calls=list(q.calls), interval=q.iv * SEC, tmin=tmin, tmax=tmax, offset=offset, filter=list(q.flt) if q.flt else None,
              flags=q.flags)
    sg, ng = tagset_map(shape, case.n)
    kw.update(group="series") if sg is None else kw.update(group="map", series_group=sg, n_groups=ng)
    kw.update(extra)
    return kw


def _refs(case, shape, qs):
    """oracle answers of the queries not answered yet, on the host's threads at once (the oracle's ctypes calls let go of the GIL)"""
    todo = [q for q in dict.fromkeys(qs) if (shape, q) not in case.refs]
    if not todo:
        return
    handles = [AggQuery(case.sh, **_kw(case, shape, q)) for q in todo]
    try:
        with ThreadPoolExecutor(THREADS) as ex:
            for q, r in zip(todo, ex.map(lambda h: oracle.scan(case.sd, h.desc, threads=1), handles)):
                case.refs[(shape, q)] = r
    finally:
        for h in handles:
            h.close()


def _same(got, want, label):
    """two dense records bitwise: validity, and values and selector times on the valid cells"""
    assert (got["n_groups"], got["n_buckets"], got["start"]) == (want["n_groups"], want["n_buckets"], want["start"]), label
    for k, (g, w) in enumerate(zip(got["cols"], want["cols"])):
        ok = np.asarray(w["valid"]) != 0
        assert np.array_equal(np.asarray(g["valid"]) != 0, ok), f"{label} call {k}: validity"
        assert np.array_equal(np.asarray(g["values"]).view(np.uint64)[ok], np.asarray(w["values"]).view(np.uint64)[ok]), f"{label} call {k}: values"
        assert (g["times"] is None) == (w["times"] is None), f"{label} call {k}: times presence"
        if w["times"] is not None:
            assert np.array_equal(np.asarray(g["times"])[ok], np.asarray(w["times"])[ok]), f"{label} call {k}: times"


def _query(case, shape, q, monkeypatch, **extra):
    """create and run q (OGPU_NO_COLS as q asks); returns the handle"""
    with monkeypatch.context() as m:
        if q.no_cols:
            m.setenv("OGPU_NO_COLS", "1")
        return AggQuery(case.sh, **_kw(case, shape, q, **extra)).run()


def _run(case, shape, q, monkeypatch, label):
    """q under the map `shape`: the path, the oracle bitwise, rows_decoded and page_bytes.  Returns the dense record."""
    ref = case.refs[(shape, q)]
    h = _query(case, shape, q, monkeypatch)
    try:
        st = h.stats()
        lab = f"{label} {case.name} {shape} {q}"
        assert st["path"] == q.path, f"{lab}: path {st['path']}"
        if q.path == 2:
            assert st["il_state"] == 1, lab
        d = h.dense_host()
        compare_dense(d, ref, q.calls, len(q.calls) > 1, lab)
        assert (st["rows_decoded"], st["page_bytes"]) == (ref["rows_decoded"], ref["page_bytes"]), lab
        return d
    finally:
        h.close()


# ---------------------------------------------------------------------------------------------------------------
# maps x paths
# ---------------------------------------------------------------------------------------------------------------
REGULAR_SHAPES = ["identity", "one", "empty_edges", "sparse", "batch_contig", "batch_strided", "permuted", "big_singletons", "series"]
RAGGED_SHAPES = ["identity", "one", "empty_edges", "permuted", "series"]
CASES = [("regular", s) for s in REGULAR_SHAPES] + [("ragged", s) for s in RAGGED_SHAPES] + [("big", "thousands"), ("big", "series")]


@pytest.mark.parametrize("name,shape", CASES, ids=[f"{a}-{b}" for a, b in CASES])
def test_every_path_under_the_map(cases, name, shape, monkeypatch):
    """every query of QUERIES under the map: paths 0, 1, 2, 4 and 5, the oracle bitwise.  The identity map also equals per-series
    output, and one tagset equals OG_GROUP_ALL under OG_Q_STRICT_ORDER, bitwise and on the same path"""
    case = _case(cases, name)
    _refs(case, shape, QUERIES)
    for q in QUERIES:
        d = _run(case, shape, q, monkeypatch, "paths")
        if shape in ("identity", "one"):
            h = _query(case, shape, q, monkeypatch, **(dict(group="series") if shape == "identity" else
                                                        dict(group="all", flags=q.flags | L.Q_STRICT_ORDER)))
            assert h.stats()["path"] == q.path, f"{shape} twin of {q}"
            _same(h.dense_host(), d, f"{case.name} {shape} twin of {q}")
            h.close()


@pytest.mark.parametrize("chunk", ["32", "96", "4096"])
@pytest.mark.parametrize("name", ["regular", "ragged"])
def test_chunk_plans_cut_tagsets(cases, name, chunk, monkeypatch):
    """OGPU_CHUNK_SERIES 32, 96 and 4096 (one chunk of the 600 or 192 series): a tagset's members sit before series_begin and
    after series_end of a chunk, so k_merge_groups finds the first one in the chunk and folds the rest chunk after chunk.  On the
    ragged shard, per-series output takes the branch for chunks whose series hold no segment (series 64..127)."""
    monkeypatch.setenv("OGPU_CHUNK_SERIES", chunk)
    case = _case(cases, name)
    for shape in (REGULAR_SHAPES if name == "regular" else RAGGED_SHAPES):
        qs = PATH_QUERIES + ([QUERIES[4]] if name == "ragged" else [])
        _refs(case, shape, qs)
        for q in qs:
            _run(case, shape, q, monkeypatch, f"chunks of {chunk}")


@pytest.mark.parametrize("chunk", ["32", "96", "4096"])
def test_thousands_of_tagsets_under_chunk_plans(cases, chunk, monkeypatch):
    """1500 tagsets over 4500 series: chunks of 32 and 96 cut two OG_IL_SUPER blocks of lane groups, chunks of 4096 give each
    block its own chunk; path 2 (all six calls) and path 5"""
    monkeypatch.setenv("OGPU_CHUNK_SERIES", chunk)
    case = _case(cases, "big")
    qs = [QUERIES[0], QUERIES[12]]
    _refs(case, "thousands", qs)
    for q in qs:
        _run(case, "thousands", q, monkeypatch, f"chunks of {chunk}")


# ---------------------------------------------------------------------------------------------------------------
# records
# ---------------------------------------------------------------------------------------------------------------
RECORD_QUERIES = [QUERIES[12], QUERIES[3], QUERIES[2], QUERIES[9], QUERIES[11]]  # RecMeta.Times; selector times; no interval; bool


@pytest.mark.parametrize("name,shape", [("regular", s) for s in ("identity", "empty_edges", "sparse", "permuted", "series")] +
                         [("ragged", s) for s in ("empty_edges", "series")])
def test_records_slice_the_dense_record(cases, name, shape, monkeypatch):
    """og_query_next drained at chunk_size 1, 7 and 1024, ascending and descending, equals the TransIntervalRec2Rec model of the
    dense record: no record for an empty tagset or window, the right group ids, sids under per-series output (series without
    segments included), RecMeta.Times of multi-call first / last, a single-call selector's point time, time 0 without an interval"""
    case = _case(cases, name)
    _refs(case, shape, RECORD_QUERIES)
    sg, ng = tagset_map(shape, case.n)
    for q in RECORD_QUERIES:
        for ascending in (True, False):
            for chunk in (1, 7, 1024):
                lab = f"records {case.name} {shape} {q} asc={ascending} chunk={chunk}"
                h = _query(case, shape, q, monkeypatch, ascending=ascending, chunk_size=chunk)
                d = h.dense_host()
                compare_dense(d, case.refs[(shape, q)], q.calls, len(q.calls) > 1, lab)
                recs = list(h.records())
                h.close()
                want = records_of(d, q.calls, ascending, chunk)
                assert_records(recs, want, lab, sids=case.sids if sg is None else None)
                members = np.bincount(sg, minlength=ng) if sg is not None else np.ones(case.n, int)
                assert all(members[r["group"]] for r in recs), f"{lab}: a record of an empty tagset"


# ---------------------------------------------------------------------------------------------------------------
# a shard without series
# ---------------------------------------------------------------------------------------------------------------
def test_a_shard_without_series():
    """og_shard_open accepts n_series = 0.  Per-series output then has one tagset with one empty window: nothing valid, and
    og_query_next at OG_EOF at once, run after run.  A map over no series and one tagset answer as the oracle does.  Before each
    query, a query of the same shape whose one cell is valid is run on a one-series shard and closed, so the device memory pool
    hands the zero-series query buffers that held valid cells: a dense record no kernel writes would show them."""
    args = (np.zeros(1, np.uint8), [], [0], [], [], [("v", L.TYPE_FLOAT, [], []), ("i", L.TYPE_INT, [], [])], [], [])
    sh, sd = Shard.open(*args), Shard.desc(*args)
    one = Shard.synth(1, 100, [(L.TYPE_FLOAT, L.SYNTH_F_HI, 0), (L.TYPE_INT, L.SYNTH_INT_WALK, 0)], t0=T0, dt=SEC, seed=3)
    assert sh.info()["n_series"] == 0
    try:
        for calls in ([("sum", 0), ("count", 1), ("last", 0)], [("max", 0)], [("first", 1)]):
            for group, kw in (("series", {}), ("map", dict(series_group=np.zeros(0, np.uint32), n_groups=3)), ("all", {})):
                for iv in (60 * SEC, 0):
                    lab = f"{calls} {group} iv={iv}"
                    primer = AggQuery(one, calls, 3600 * SEC if iv else 0, T0, T0 + 99 * SEC, group="series").run()
                    assert all(np.asarray(c["valid"]).all() for c in primer.dense_host()["cols"]), lab
                    primer.close()
                    q = AggQuery(sh, calls, iv, T0, T0 + 3600 * SEC, group=group, **kw)
                    for _ in range(2):
                        q.run()
                        d = q.dense_host()
                        assert (d["n_groups"], d["n_buckets"]) == ({"series": 1, "all": 1, "map": 3}[group], 1), lab
                        for c in d["cols"]:
                            assert not np.asarray(c["valid"]).any(), lab
                        if group != "series":  # the oracle has no tagset for per-series output over no series
                            compare_dense(d, oracle.scan(sd, q.desc, threads=1), calls, len(calls) > 1, lab)
                        assert list(q.records()) == [], lab
                        st = q.stats()
                        assert (st["rows_decoded"], st["page_bytes"], st["segments_scanned"]) == (0, 0, 0), lab
                    q.close()
    finally:
        sh.close()
        one.close()


# ---------------------------------------------------------------------------------------------------------------
# refusals
# ---------------------------------------------------------------------------------------------------------------
def test_bad_maps_are_refused_and_the_shard_still_answers(cases, monkeypatch):
    """og_query_create: OG_E_INVAL for a series_group entry equal to n_groups, for n_groups = 0 and for a NULL series_group"""
    case = _case(cases, "regular")
    q = QUERIES[0]
    _refs(case, "permuted", [q])
    good = AggQuery(case.sh, **_kw(case, "permuted", q))
    sg, ng = tagset_map("permuted", case.n)
    over = sg.copy()
    over[case.n // 2] = ng
    for label, edit in (("entry == n_groups", lambda d: setattr(d, "series_group", over.ctypes.data_as(C.POINTER(C.c_uint32)))),
                        ("n_groups == 0", lambda d: setattr(d, "n_groups", 0)),
                        ("NULL series_group", lambda d: setattr(d, "series_group", None))):
        d = L.QueryDesc.from_buffer_copy(good.desc)
        edit(d)
        h = C.c_void_p()
        assert L.lib().og_query_create(case.sh.h, C.byref(d), C.byref(h)) == L.OG_E_INVAL, label
        assert not h.value, label
        _run(case, "permuted", q, monkeypatch, f"after refusing {label}")
    good.close()
