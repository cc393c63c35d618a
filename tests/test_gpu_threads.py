"""The header's thread promises: distinct queries may run concurrently, and og_query_create on another thread waits while an
append or a compaction runs.

ctypes releases the GIL around every library call, so these threads run the library concurrently.  Every thread starts at a
threading.Barrier, is a daemon, and is joined with a timeout that fails the test; each scenario runs once.  Every concurrent answer
is compared bit for bit with the same query run alone.  No environment variable is set here: the library reads some while it
plans a query."""
import threading

import numpy as np
import pytest

import oracle
from opengemini_b200 import AggQuery, Shard
from opengemini_b200 import _lib as L
from test_gpu_compact import _synth_with_flushes
from test_gpu_out_of_order import SEC, T0

pytestmark = pytest.mark.gpu
COLS = [(L.TYPE_FLOAT, L.SYNTH_F_HI, 0), (L.TYPE_FLOAT, L.SYNTH_F_LO, 0), (L.TYPE_INT, L.SYNTH_INT_WALK, 0), (L.TYPE_BOOL, L.SYNTH_BOOL, 0)]
N_SERIES, ROWS = 64, 3000
TMAX = T0 + (ROWS - 1) * SEC
JOIN_S = 300


@pytest.fixture(scope="module", autouse=True)
def _device():
    Shard.init(0)


def _queries(f):
    """(calls, kwargs, og_stats.path) on float column f of a regular shard: every aggregate path"""
    fc = [("sum", f), ("count", f), ("max", f)]
    two = [("sum", f), ("sum", 2)]
    return [(fc, dict(), 3),
            (fc, dict(flags=L.Q_STRICT_ORDER), 2),
            (fc, dict(flags=L.Q_NO_FAST), 1),
            (fc, dict(flags=L.Q_NO_FUSED | L.Q_STRICT_ORDER), 0),
            (two, dict(filter=[("term", f, ">", 100.0)], flags=L.Q_STRICT_ORDER), 5),
            (two, dict(filter=[("term", f, ">", 100.0), ("term", 2, "<", 0), "and"], flags=L.Q_STRICT_ORDER), 4)]


def _answer(sh, calls, kw, tmax=TMAX, chunk_size=1024):
    """create, run, read and destroy one query: (dense cells, og_query_next records, stats)"""
    q = AggQuery(sh, calls, 60 * SEC, T0, tmax, chunk_size=chunk_size, **kw).run()
    d = q.dense_host()
    dense = (d["n_groups"], d["n_buckets"], d["start"],
             [(c["valid"].tobytes(), c["values"].tobytes(), None if c["times"] is None else c["times"].tobytes()) for c in d["cols"]])
    recs = [_rec_bytes(r) for r in q.records()]
    st = q.stats()
    q.close()
    return dense, recs, st


def _rec_bytes(r):
    return (r["rows"], r["group"], r["sid"], r["times"].tobytes(),
            [(c["valid"].tobytes(), c["values"].tobytes(), None if c["times"] is None else c["times"].tobytes()) for c in r["cols"]])


def _run_threads(targets):
    """start every target at one barrier, as daemon threads; join each with a timeout; re-raise the first failure"""
    barrier = threading.Barrier(len(targets))
    out, errors = [None] * len(targets), []

    def body(i, fn):
        try:
            barrier.wait(timeout=JOIN_S)
            out[i] = fn()
        except BaseException as e:  # noqa: BLE001 - reported on the main thread
            errors.append(e)

    threads = [threading.Thread(target=body, args=(i, fn), daemon=True) for i, fn in enumerate(targets)]
    for t in threads:
        t.start()
    for t in threads:
        t.join(timeout=JOIN_S)
        assert not t.is_alive(), "a thread did not finish: deadlock or hang"
    if errors:
        raise errors[0]
    return out


def test_concurrent_first_queries_build_each_copy_once():
    """Four threads start together on a shard without interleaved copies, two on each float column, so the two builds of each
    copy race; two threads begin with queries that do not build the copy (paths 1 and 0) while the others build it.  Every dense
    cell and record equals the same query run alone afterwards, bit for bit; the copy is built once, as large as a single-threaded
    build on an identical shard; and no query reports a copy that another thread is still building."""
    sh = Shard.synth(N_SERIES, ROWS, COLS, t0=T0, dt=SEC, seed=17)
    twin = Shard.synth(N_SERIES, ROWS, COLS, t0=T0, dt=SEC, seed=17)
    plans = []
    for k in range(4):
        qs = _queries(k // 2)
        plans.append(qs if k % 2 == 0 else qs[2:] + qs[:2])   # threads 1 and 3 start on paths 1, 0, 5, 4

    def work(qs):
        return [_answer(sh, calls, kw) for calls, kw, _p in qs]

    got = _run_threads([lambda qs=qs: work(qs) for qs in plans])
    alone_bytes = {}
    for f in (0, 1):
        st = _answer(twin, *_queries(f)[0][:2])[2]
        assert st["il_state"] == 1 and st["path"] == 3
        alone_bytes[f] = st["il_bytes"]
    for k, qs in enumerate(plans):
        f = k // 2
        for (calls, kw, path), (dense, recs, st) in zip(qs, got[k]):
            alone = _answer(sh, calls, kw)
            assert dense == alone[0], (k, calls, kw)
            assert recs == alone[1], (k, calls, kw)
            assert st["path"] == path, (k, calls, kw, st["path"])
            if path in (3, 2):  # these queries built the copy, or waited for the thread that did
                assert st["il_state"] == 1 and st["il_bytes"] == alone_bytes[f], (k, path, st["il_state"], st["il_bytes"])
            elif path in (1, 0):  # not built yet, or ready: never the -1 of a build in progress
                assert st["il_state"] in (0, 1), (k, path, st["il_state"])
    for f in (0, 1):
        st = _answer(sh, *_queries(f)[0][:2])[2]
        assert st["il_state"] == 1 and st["il_bytes"] == alone_bytes[f]
    sh.close(); twin.close()


def test_queries_of_two_shards_on_two_threads():
    """Two threads query two shards and take turns at og_query_next, record by record: each query's records equal its records
    when it runs alone."""
    a = Shard.synth(N_SERIES, ROWS, COLS, t0=T0, dt=SEC, seed=21)
    b = Shard.synth(N_SERIES // 2, ROWS + 500, COLS, t0=T0, dt=SEC, seed=22)
    kw_a = dict(group="series", flags=L.Q_STRICT_ORDER)
    kw_b = dict(filter=[("term", 1, ">", 20.0)], group="series", flags=L.Q_STRICT_ORDER)
    calls_a, calls_b = [("sum", 0), ("max", 0), ("first", 2)], [("count", 1), ("min", 2)]
    tmax_b = T0 + (ROWS + 499) * SEC
    want_a = _answer(a, calls_a, kw_a, chunk_size=64)[1]
    want_b = _answer(b, calls_b, kw_b, tmax=tmax_b, chunk_size=64)[1]
    turns = min(len(want_a), len(want_b))
    assert turns > 10
    step = threading.Barrier(2)

    def drain(sh, calls, kw, tmax):
        q = AggQuery(sh, calls, 60 * SEC, T0, tmax, chunk_size=64, **kw).run()
        it, recs = q.records(), []
        for _ in range(turns):  # one og_query_next per turn, the other thread's between
            step.wait(timeout=JOIN_S)
            recs.append(_rec_bytes(next(it)))
        recs += [_rec_bytes(r) for r in it]
        q.close()
        return recs

    got_a, got_b = _run_threads([lambda: drain(a, calls_a, kw_a, TMAX), lambda: drain(b, calls_b, kw_b, tmax_b)])
    assert got_a == want_a
    assert got_b == want_b
    a.close(); b.close()


def _flush_desc(seed, first_row, rows):
    src = Shard.synth(16, rows, COLS[:3], t0=T0 + first_row * SEC, dt=SEC, seed=seed)
    d = oracle.shard_desc_from_export(src.export())
    src.close()
    return d


@pytest.mark.parametrize("mutation", ["append", "compact"])
def test_create_against_a_mutation(mutation):
    """Thread A appends a flush (or compacts) while thread B creates, runs and destroys one query, both from one barrier.  A
    succeeds, or is refused with OG_E_STATE because B's query was alive first and then succeeds after the join; B's answer is,
    bit for bit, the answer before the mutation or the one after it, both computed on one thread."""
    if mutation == "append":
        sh = Shard.synth(16, 2000, COLS[:3], t0=T0, dt=SEC, seed=31)
        twin = Shard.synth(16, 2000, COLS[:3], t0=T0, dt=SEC, seed=31)
        flush = _flush_desc(32, 2000, 700)
        mutate = lambda s_: s_.append_files([(flush, False)])  # noqa: E731
    else:
        sh = _synth_with_flushes(16, 2000, 4, 90, seed=33)
        twin = _synth_with_flushes(16, 2000, 4, 90, seed=33)
        mutate = lambda s_: s_.compact()  # noqa: E731
    tmax = T0 + 3000 * SEC
    queries = [([("sum", 0), ("count", 0), ("max", 0)], dict()), ([("sum", 0), ("last", 1), ("min", 2)], dict(group="series"))]
    before = [_answer(sh, calls, kw, tmax)[:2] for calls, kw in queries]
    _answer(sh, *queries[0], tmax)  # the interleaved copy exists when the mutation starts
    mutate(twin)
    after = [_answer(twin, calls, kw, tmax)[:2] for calls, kw in queries]
    assert before[0] != after[0]
    for k, (calls, kw) in enumerate(queries):
        def mutator():
            try:
                mutate(sh)
                return L.OG_OK
            except L.OgpuError as e:
                assert e.status == L.OG_E_STATE, str(e)
                return e.status

        status, got = _run_threads([mutator, lambda: _answer(sh, calls, kw, tmax)[:2]])
        if status == L.OG_E_STATE:
            mutate(sh)
        assert got == before[k] or got == after[k], (mutation, k)
        assert [_answer(sh, c, w, tmax)[:2] for c, w in queries] == after
        if k + 1 < len(queries):  # the next round starts from the shard before the mutation
            sh.close()
            sh = Shard.synth(16, 2000, COLS[:3], t0=T0, dt=SEC, seed=31) if mutation == "append" else _synth_with_flushes(16, 2000, 4, 90, seed=33)
            _answer(sh, *queries[0], tmax)
    sh.close(); twin.close()
