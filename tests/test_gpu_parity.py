"""GPU parity tests (need an H100): the CUDA path, called through the C ABI, against the CPU oracle.

Bar: bit-exact for everything, including float sums when the query asks for OG_Q_STRICT_ORDER — the kernels then keep
the reference's summation order (left-to-right inside a record window, prev+curr across records, series order across
series).  Without the flag a one-tagset query folds the 32 series of a lane group with warp shuffles first: counts,
min/max/first/last and their times are still compared bitwise, float sums to 1e-12 relative (north_star allows 1e-9).
run_both() runs every one-tagset query both ways.
"""
import ctypes as C
import struct

import numpy as np
import pytest

import oracle
from opengemini_b200 import AggQuery, Shard
from opengemini_b200 import _lib as L

pytestmark = pytest.mark.gpu

T0 = 1_700_000_000_000_000_000
SEC = 1_000_000_000


@pytest.fixture(scope="module", autouse=True)
def _device():
    Shard.init(0)


def _bits(t):
    a = t.cpu().numpy() if hasattr(t, "cpu") else np.asarray(t)
    return a.view(np.uint64) if a.dtype != np.uint64 else a


SUM_RTOL = 1e-12


def compare_dense(gpu, ref, calls, multi, label="", float_sum_exact=True, col_types=None):
    assert gpu["n_groups"] == ref["n_groups"] and gpu["n_buckets"] == ref["n_buckets"], label
    assert gpu["start"] == ref["start"], label
    for k, (func, _col) in enumerate(calls):
        g, r = gpu["cols"][k], ref["cols"][k]
        gv = np.asarray(g["valid"]).astype(bool)
        rv = r["valid"].astype(bool)
        assert np.array_equal(gv, rv), f"{label} call {k} ({func}): validity differs at {np.flatnonzero(gv != rv)[:5]}"
        gb, rb = _bits(g["values"])[rv], r["values"][rv]
        if func == "sum" and not float_sum_exact and g["type"] == L.TYPE_FLOAT:
            gf, rf = gb.view(np.float64), rb.view(np.float64)
            err = np.abs(gf - rf) / np.maximum(np.abs(rf), 1e-300)
            assert np.all((err <= SUM_RTOL) | (gf == rf)), f"{label} call {k} (sum): folded sums off by {err.max():.3e} relative"
            continue
        bad = np.flatnonzero(gb != rb)
        assert bad.size == 0, f"{label} call {k} ({func}): {bad.size} value cells differ, first at valid-index {bad[:3]}: gpu={gb[bad[:3]]} ref={rb[bad[:3]]}"
        carries_time = func in ("min", "max", "first", "last") and not (multi and func in ("min", "max"))
        if carries_time:
            assert g["times"] is not None, f"{label} call {k}: missing times"
            gt, rt = np.asarray(g["times"])[rv], r["times"][rv]
            assert np.array_equal(gt, rt), f"{label} call {k} ({func}): row times differ"


def run_both(shard, shard_desc, calls, interval, tmin, tmax, label, flags=0, folded=True, **kw):
    """strict order: everything bitwise.  Then, for one-tagset queries on the fused path, the default (folded) order
    (folded=False skips it: with NaN partials the reference's own cross-series update depends on the series order)."""
    q = AggQuery(shard, calls, interval, tmin, tmax, flags=flags | L.Q_STRICT_ORDER, **kw).run()
    gpu = q.dense_host()
    ref = oracle.scan(shard_desc, q.desc, threads=1)
    compare_dense(gpu, ref, calls, len(calls) > 1, label)
    st = q.stats()
    assert st["rows_decoded"] == ref["rows_decoded"], label
    assert st["page_bytes"] == ref["page_bytes"], label
    assert st["path"] != 3, label
    q.close()
    if folded and kw.get("group", "all") == "all" and not (flags & (L.Q_NO_FUSED | L.Q_NO_FAST)):
        q2 = AggQuery(shard, calls, interval, tmin, tmax, flags=flags, **kw).run()
        compare_dense(q2.dense_host(), ref, calls, len(calls) > 1, label + " [folded]", float_sum_exact=False)
        q2.run()  # second run of the same plan: scratch reuse (cell validity is only cleared after a run that used the cells)
        compare_dense(q2.dense_host(), ref, calls, len(calls) > 1, label + " [folded, rerun]", float_sum_exact=False)
        q2.close()
    return gpu, ref


# ---------------------------------------------------------------------------------------------------------------
# K7: device encoders == restated reference encoders, byte for byte
# ---------------------------------------------------------------------------------------------------------------
SYNTH_COLS = [(L.TYPE_FLOAT, L.SYNTH_F_HI, 0), (L.TYPE_FLOAT, L.SYNTH_F_LO, 0), (L.TYPE_INT, L.SYNTH_INT_WALK, 0),
              (L.TYPE_BOOL, L.SYNTH_BOOL, 0), (L.TYPE_FLOAT, L.SYNTH_F_HI, 50), (L.TYPE_INT, L.SYNTH_INT_WALK, 50),
              (L.TYPE_BOOL, L.SYNTH_BOOL, 300), (L.TYPE_FLOAT, L.SYNTH_F_LO, 1000)]


@pytest.mark.parametrize("rows", [2500, 1000, 1001, 7])
def test_synth_pages_byte_exact(rows):
    hs = oracle.HostShard(5, rows, SYNTH_COLS, t0=T0, dt=SEC, seed=42)
    gs = Shard.synth(5, rows, SYNTH_COLS, t0=T0, dt=SEC, seed=42)
    ex = gs.export()
    nseg = ex["seg_tmin"].size
    assert nseg == hs.desc.n_segments
    assert np.array_equal(ex["seg_tmin"], np.ctypeslib.as_array(hs.desc.seg_tmin, shape=(nseg,)))
    assert np.array_equal(ex["seg_tmax"], np.ctypeslib.as_array(hs.desc.seg_tmax, shape=(nseg,)))
    for c in range(len(SYNTH_COLS) + 1):
        for g in range(nseg):
            off, ln = int(ex["page_off"][c, g]), int(ex["page_len"][c, g])
            got = ex["data"][off:off + ln]
            want = hs.page(c, g)
            assert got.size == want.size and np.array_equal(got, want), \
                f"column {c} segment {g}: device page ({got.size} B, head {got[:12]}) != oracle page ({want.size} B, head {want[:12]})"
    gs.close()


# ---------------------------------------------------------------------------------------------------------------
# K1-K4/K6: materialise path
# ---------------------------------------------------------------------------------------------------------------
def test_decode_segment_matches_oracle():
    hs = oracle.HostShard(3, 2300, SYNTH_COLS, t0=T0, dt=SEC, seed=7)
    sh = Shard.open_desc(hs.desc, keepalive=hs)
    for seg in range(hs.desc.n_segments):
        rec = sh.decode_segment(seg)
        want_t = oracle.time_page_decode(hs.page(len(SYNTH_COLS), seg))
        assert np.array_equal(rec["times"], want_t)
        for c, (typ, _d, _n) in enumerate(SYNTH_COLS):
            wv, wvalid = oracle.field_page_decode(typ, hs.page(c, seg))
            col = rec["cols"][c]
            assert col["len"] == wvalid.size and col["nil_count"] == int((~wvalid).sum())
            assert np.array_equal(col["valid"], wvalid), f"seg {seg} col {c} bitmap"
            assert np.array_equal(col["values"].view(np.uint8), wv.view(np.uint8)), f"seg {seg} col {c} values"
    sh.close()


def _one_segment_shard(typ, page, time_page, rows_t, n_cols=1):
    """n_cols > 1: every column reads the same page"""
    data = np.concatenate([page, time_page])
    cols = [(f"v{c}", typ, [0], [page.size]) for c in range(n_cols)]
    return Shard.open(data, [1], [0, 1], [rows_t[0]], [rows_t[-1]], cols, [page.size], [time_page.size])


@pytest.mark.parametrize("shape", ["raw", "same", "same0", "rle", "rle0", "gorilla", "gorilla_wrap", "one", "empty", "nulls"])
def test_float_codecs_decode(shape):
    rng = np.random.default_rng(3)
    n = 1000
    valid = None
    if shape == "raw":
        v = rng.integers(0, 2**63, n).view(np.float64)
        v = np.where(np.isfinite(v), v, 1.0)
    elif shape == "same":
        v = np.full(n, 3.25)
    elif shape == "same0":
        v = np.zeros(n)
    elif shape == "rle":
        v = np.repeat([1.5, 2.5, 0.0, 7.0], n // 4)
    elif shape == "rle0":
        v = np.repeat([0.0, 4.0, 0.0, 0.0, 9.0], n // 5)
    elif shape == "gorilla":
        v = 100 + rng.random(n)
    elif shape == "gorilla_wrap":
        v = (np.uint64(0x4059000000000000) + rng.integers(0, 1000, n).astype(np.uint64)).view(np.float64)
    elif shape == "one":
        v = np.array([42.5]); n = 1
    elif shape == "empty":
        v = np.zeros(n); valid = np.zeros(n, np.uint8)
    else:
        v = 100 + rng.random(n); valid = (rng.random(n) > 0.1).astype(np.uint8)
    page = oracle.field_page_encode(L.TYPE_FLOAT, v, valid)
    t = T0 + np.arange(n, dtype=np.int64) * SEC
    sh = _one_segment_shard(L.TYPE_FLOAT, page, oracle.time_page_encode(t), t)
    rec = sh.decode_segment(0)
    wv, wvalid = oracle.field_page_decode(L.TYPE_FLOAT, page)
    assert np.array_equal(rec["cols"][0]["valid"], wvalid)
    assert np.array_equal(rec["cols"][0]["values"].view(np.uint64), wv.view(np.uint64))
    sh.close()


@pytest.mark.parametrize("shape", ["const", "s8b", "s8b_ones", "raw2", "bigdelta", "nulls"])
def test_int_codecs_decode(shape):
    rng = np.random.default_rng(5)
    n = 1000
    valid = None
    if shape == "const":
        v = np.arange(n, dtype=np.int64) * -7 + 3
    elif shape == "s8b":
        v = np.cumsum(rng.integers(-1000, 1001, n)).astype(np.int64)
    elif shape == "s8b_ones":
        v = -np.arange(n, dtype=np.int64); v[-1] += 5
    elif shape == "raw2":
        v = np.array([5, -9], np.int64); n = 2
    elif shape == "bigdelta":
        v = np.where(np.arange(n) % 2 == 0, 1 << 40, -(1 << 40)).astype(np.int64)
    else:
        v = np.cumsum(rng.integers(-50, 51, n)).astype(np.int64); valid = (rng.random(n) > 0.2).astype(np.uint8)
    page = oracle.field_page_encode(L.TYPE_INT, v, valid)
    t = T0 + np.arange(n, dtype=np.int64) * SEC
    sh = _one_segment_shard(L.TYPE_INT, page, oracle.time_page_encode(t), t)
    rec = sh.decode_segment(0)
    wv, wvalid = oracle.field_page_decode(L.TYPE_INT, page)
    assert np.array_equal(rec["cols"][0]["valid"], wvalid)
    assert np.array_equal(rec["cols"][0]["values"], wv)
    sh.close()


@pytest.mark.parametrize("shape", ["const", "s8b_scaled", "s8b_unscaled", "raw2", "one"])
def test_time_codecs_decode(shape):
    rng = np.random.default_rng(9)
    if shape == "const":
        t = T0 + np.arange(1000, dtype=np.int64) * SEC
    elif shape == "s8b_scaled":
        t = T0 + np.cumsum(rng.integers(1, 50, 1000) * 1_000_000).astype(np.int64)
    elif shape == "s8b_unscaled":
        t = T0 + np.cumsum(rng.integers(1, 5000, 777)).astype(np.int64)
    elif shape == "raw2":
        t = np.array([T0, T0 + 17], np.int64)
    else:
        t = np.array([T0 + 5], np.int64)
    v = 100 + rng.random(t.size)  # full-mantissa values: Gorilla (few-decimal values would route to Snappy, float.go:206)
    page = oracle.field_page_encode(L.TYPE_FLOAT, v)
    sh = _one_segment_shard(L.TYPE_FLOAT, page, oracle.time_page_encode(t), t)
    rec = sh.decode_segment(0)
    assert np.array_equal(rec["times"], t)
    # and through the fused + generic aggregate paths: irregular time pages drive the TimeIter
    for flags in (0, L.Q_NO_FUSED):
        q = AggQuery(sh, [("sum", 0), ("count", 0), ("max", 0)], 7 * SEC, int(t[0]), int(t[-1]), flags=flags).run()
        d = q.dense_host()
        b = (t - d["start"]) // (7 * SEC)
        want_cnt = np.bincount(b, minlength=d["n_buckets"])
        assert np.array_equal(d["cols"][1]["values"] * d["cols"][1]["valid"], want_cnt)
        q.close()
    sh.close()


def test_unsupported_and_corrupt_pages_fail_cleanly():
    n = 100
    t = T0 + np.arange(n, dtype=np.int64) * SEC
    tp = oracle.time_page_encode(t)
    good = oracle.field_page_encode(L.TYPE_FLOAT, 100 + np.random.default_rng(1).random(n))
    for tag, want in ((0x20, L.OG_E_CORRUPT), (0x60, L.OG_E_UNSUPPORTED), (0x70, L.OG_E_CORRUPT)):  # 0x20: Snappy tag over Gorilla bytes = a corrupt Snappy block
        bad = good.copy(); bad[5] = tag  # block tag byte after the 5-byte Full header
        with pytest.raises(L.OgpuError) as ei:
            _one_segment_shard(L.TYPE_FLOAT, bad, tp, t)
        assert ei.value.status == want
    ipage = oracle.field_page_encode(L.TYPE_INT, np.arange(n, dtype=np.int64) ** 2)
    bad = ipage.copy(); bad[5] = 0x30  # zstd
    with pytest.raises(L.OgpuError) as ei:
        _one_segment_shard(L.TYPE_INT, bad, tp, t)
    assert ei.value.status == L.OG_E_UNSUPPORTED
    # type mismatch on a page with a normal (partial-null) header
    valid = np.ones(n, np.uint8); valid[3] = 0
    fpage = oracle.field_page_encode(L.TYPE_FLOAT, np.ones(n), valid)
    with pytest.raises(L.OgpuError) as ei:
        _one_segment_shard(L.TYPE_INT, fpage, tp, t)
    assert ei.value.status == L.OG_E_TYPE
    # a call on a column that does not exist is rejected, not mis-executed
    sh = _one_segment_shard(L.TYPE_FLOAT, good, tp, t)
    d = L.QueryDesc(); calls = (L.Call * 1)(); calls[0].func, calls[0].column = L.AGG_SUM, 7
    d.interval, d.tmin, d.tmax, d.ascending, d.n_calls, d.calls = SEC, int(t[0]), int(t[-1]), 1, 1, calls
    h = C.c_void_p()
    assert L.lib().og_query_create(sh.h, C.byref(d), C.byref(h)) == L.OG_E_INVAL
    sh.close()


def _be(fmt, *v):
    return np.frombuffer(struct.pack(">" + fmt, *v), np.uint8)


def test_payload_that_disagrees_with_the_value_count(monkeypatch):
    """Pages that pass og_shard_open but whose words / runs / bit stream do not hold the header's value count fail the same way
    on every generic decode path; zero-length RLE runs of zeros pad nothing, zero-length runs of a value are corrupt.  A page whose
    validity bitmap disagrees with its nil count is refused at og_shard_open."""
    n = 100
    t = T0 + np.arange(n, dtype=np.int64) * SEC
    tp = oracle.time_page_encode(t)
    ipage = oracle.field_page_encode(L.TYPE_INT, np.cumsum(np.random.default_rng(2).integers(-1000, 1001, n)).astype(np.int64))
    assert ipage[5] >> 4 == 2  # Full header (5 B), then [tag][u32 encCount][u32 srcCount][u64 first][encCount - 1 words]
    enc = struct.unpack(">I", ipage[6:10].tobytes())[0]
    assert ipage.size == 14 + 8 * enc
    surplus = np.concatenate([ipage[:6], _be("I", enc + 1), ipage[10:], _be("Q", 0xF << 60)])  # one more word: selector 15, one value
    missing = np.concatenate([ipage[:6], _be("I", enc - 1), ipage[10:-8]])
    fpage = oracle.field_page_encode(L.TYPE_FLOAT, np.repeat([1.5, 2.5, 0.0, 7.0], n // 4))
    assert fpage[5] >> 4 == 5  # RLE: runs of [u16 BE count (bit 15: zero run)][8 B LE value]
    run0 = struct.unpack(">H", fpage[6:8].tobytes())[0]
    rle_n1 = np.concatenate([fpage[:6], _be("H", run0 + 1), fpage[8:]])
    rle_zero0 = np.concatenate([fpage[:6], _be("H", 0x8000), fpage[6:]])
    rle_value0 = np.concatenate([fpage[:6], _be("H", 0), np.full(8, 0x11, np.uint8), fpage[6:]])
    gpage = oracle.field_page_encode(L.TYPE_FLOAT, 100 + np.random.default_rng(3).random(n))
    assert gpage[5] >> 4 == 3  # Gorilla: [tag][0x10][8 B first][bit stream]
    gorilla_cut = gpage[:15 + (gpage.size - 15) // 2]  # half the bit stream

    def paths(typ, page):
        """(label, run) for og_decode_segment and paths 1, 0, 4 and 5; run() returns the dense result of the aggregates"""
        sh = _one_segment_shard(typ, page, tp, t, n_cols=2)

        def query(calls, flags, path):
            q = AggQuery(sh, calls, 0, int(t[0]), int(t[-1]), flags=flags)
            try:
                q.run()
                assert q.stats()["path"] == path
                return q.dense_host()
            finally:
                q.close()

        def multi():
            with monkeypatch.context() as m:
                m.setenv("OGPU_NO_COLS", "1")
                return query([("sum", 0), ("count", 1), ("max", 0)], 0, 4)
        return sh, [("decode", lambda: sh.decode_segment(0)),
                    ("path 1", lambda: query([("sum", 0), ("count", 0), ("max", 0)], L.Q_NO_FAST, 1)),
                    ("path 0", lambda: query([("sum", 0), ("count", 0), ("max", 0)], L.Q_NO_FUSED, 0)),
                    ("path 4", multi),
                    ("path 5", lambda: query([("sum", 0), ("count", 1), ("max", 0)], 0, 5))]

    for label, typ, page in (("s8b surplus word", L.TYPE_INT, surplus), ("s8b missing word", L.TYPE_INT, missing),
                             ("rle n+1", L.TYPE_FLOAT, rle_n1), ("rle zero-length value run", L.TYPE_FLOAT, rle_value0),
                             ("truncated gorilla", L.TYPE_FLOAT, gorilla_cut)):
        sh, runs = paths(typ, page)
        for where, run in runs:
            with pytest.raises(L.OgpuError) as ei:
                run()
            assert ei.value.status == L.OG_E_CORRUPT, f"{label}, {where}"
        sh.close()

    want, _ = oracle.field_page_decode(L.TYPE_FLOAT, rle_zero0)
    assert want.size == n
    s = 0.0
    for x in want:
        s += x
    sh, runs = paths(L.TYPE_FLOAT, rle_zero0)
    for where, run in runs:
        got = run()
        if where == "decode":
            assert np.array_equal(got["cols"][0]["values"].view(np.uint64), want.view(np.uint64)), where
            continue
        vals = [got["cols"][k]["values"][0] for k in range(3)]
        assert all(got["cols"][k]["valid"][0] for k in range(3)), where
        assert (float(vals[0]), int(vals[1]), float(vals[2])) == (s, n, want.max()), where
    sh.close()

    # a Simple8b time page with a missing word is refused when the shard is opened
    ti = T0 + np.cumsum(np.random.default_rng(4).integers(1, 5000, n)).astype(np.int64)
    tpage = oracle.time_page_encode(ti)
    assert tpage[5] >> 4 == 2  # [tag][u64 scale][u32 encCount][u32 srcCount][u64 first][encCount - 1 words]
    tenc = struct.unpack(">I", tpage[14:18].tobytes())[0]
    assert tpage.size == 22 + 8 * tenc
    tbad = np.concatenate([tpage[:14], _be("I", tenc - 1), tpage[18:-8]])
    with pytest.raises(L.OgpuError) as ei:
        _one_segment_shard(L.TYPE_FLOAT, oracle.field_page_encode(L.TYPE_FLOAT, 100 + np.zeros(n)), tbad, ti)
    assert ei.value.status == L.OG_E_CORRUPT

    # a bitmap that marks one row more valid than the header's value count is refused when the shard is opened
    valid = np.ones(n, np.uint8); valid[[3, 50]] = 0
    npage = oracle.field_page_encode(L.TYPE_FLOAT, 100 + np.random.default_rng(5).random(n), valid)
    assert npage[0] == L.TYPE_FLOAT  # normal header: [type][u32 bitmap bytes][bitmap][u32 bitmap offset][u32 nil count][block]
    nb = struct.unpack(">I", npage[1:5].tobytes())[0]
    nil = struct.unpack(">I", npage[9 + nb:13 + nb].tobytes())[0]
    assert nil == 2
    bad = np.concatenate([npage[:9 + nb], _be("I", nil + 1), npage[13 + nb:]])
    _one_segment_shard(L.TYPE_FLOAT, npage, tp, t).close()
    with pytest.raises(L.OgpuError) as ei:
        _one_segment_shard(L.TYPE_FLOAT, bad, tp, t)
    assert ei.value.status == L.OG_E_CORRUPT


# ---------------------------------------------------------------------------------------------------------------
# K5: aggregate parity (fused and generic paths) against the reference-structured oracle
# ---------------------------------------------------------------------------------------------------------------
AGG_COLS = [(L.TYPE_FLOAT, L.SYNTH_F_HI, 0), (L.TYPE_INT, L.SYNTH_INT_WALK, 0), (L.TYPE_BOOL, L.SYNTH_BOOL, 0),
            (L.TYPE_FLOAT, L.SYNTH_F_LO, 50), (L.TYPE_INT, L.SYNTH_INT_WALK, 200), (L.TYPE_BOOL, L.SYNTH_BOOL, 100)]


@pytest.fixture(scope="module")
def agg_shard():
    hs = oracle.HostShard(7, 4321, AGG_COLS, t0=T0, dt=SEC, seed=11)
    sh = Shard.open_desc(hs.desc, keepalive=hs)
    yield sh, hs
    sh.close()


ALL6 = ["count", "sum", "min", "max", "first", "last"]


@pytest.mark.parametrize("flags", [0, L.Q_NO_FUSED], ids=["fused", "generic"])
@pytest.mark.parametrize("interval", [60 * SEC, 7 * SEC, 3600 * SEC, 0])
@pytest.mark.parametrize("col", [0, 1, 3, 4])
def test_single_call_aggregates(agg_shard, col, interval, flags):
    sh, hs = agg_shard
    tmin, tmax = T0, T0 + 4320 * SEC
    for f in ALL6:
        run_both(sh, hs.desc, [(f, col)], interval, tmin, tmax, f"{f}(col{col}) iv={interval} flags={flags}", flags=flags)


@pytest.mark.parametrize("flags", [0, L.Q_NO_FUSED], ids=["fused", "generic"])
@pytest.mark.parametrize("col", [0, 1, 3, 4])
def test_multi_call_aggregates(agg_shard, col, flags):
    sh, hs = agg_shard
    for interval in (60 * SEC, 1000 * SEC, 0):
        run_both(sh, hs.desc, [(f, col) for f in ALL6], interval, T0, T0 + 4320 * SEC, f"all6(col{col}) iv={interval}", flags=flags)
    run_both(sh, hs.desc, [("sum", col), ("count", col)], 60 * SEC, T0, T0 + 4320 * SEC, "mean", flags=flags)


@pytest.mark.parametrize("col", [2, 5])
def test_bool_aggregates(agg_shard, col):
    sh, hs = agg_shard
    for flags in (0, L.Q_NO_FUSED):
        for f in ("count", "min", "max", "first", "last"):
            run_both(sh, hs.desc, [(f, col)], 60 * SEC, T0, T0 + 4320 * SEC, f"{f}(bool{col})", flags=flags)
        run_both(sh, hs.desc, [(f, col) for f in ("count", "min", "max", "first", "last")], 90 * SEC, T0, T0 + 4320 * SEC, "bool multi", flags=flags)


@pytest.mark.parametrize("flags", [0, L.Q_NO_FUSED], ids=["fused", "generic"])
def test_time_range_and_offset(agg_shard, flags):
    sh, hs = agg_shard
    # range cutting segments in the middle, windows not aligned to the range, GROUP BY time(1m, 7s)
    run_both(sh, hs.desc, [("sum", 0), ("count", 0)], 60 * SEC, T0 + 1234 * SEC + 5, T0 + 3456 * SEC + 7, "mid-range", flags=flags)
    run_both(sh, hs.desc, [("max", 0)], 60 * SEC, T0 + 999 * SEC, T0 + 1001 * SEC, "two-row range", flags=flags)
    run_both(sh, hs.desc, [("first", 3)], 60 * SEC, T0 - 500 * SEC, T0 + 10_000 * SEC, "range wider than data", flags=flags)
    run_both(sh, hs.desc, [("sum", 1), ("last", 1)], 60 * SEC, T0, T0 + 4320 * SEC, "offset 7s", flags=flags, offset=7 * SEC)
    run_both(sh, hs.desc, [("min", 4)], 61 * SEC, T0 + 17, T0 + 4000 * SEC, "odd interval", flags=flags, offset=-13 * SEC)


@pytest.mark.parametrize("group", ["series", "map"])
def test_group_modes(agg_shard, group):
    sh, hs = agg_shard
    kw = dict(group=group)
    if group == "map":
        kw.update(series_group=[2, 0, 1, 0, 2, 2, 0], n_groups=3)
    for flags in (0, L.Q_NO_FUSED):
        for calls in ([("sum", 0), ("count", 0)], [("max", 0)], [("first", 4)], [(f, 3) for f in ALL6]):
            run_both(sh, hs.desc, calls, 60 * SEC, T0, T0 + 4320 * SEC, f"group={group} {calls}", flags=flags, **kw)


def test_where_filters(agg_shard):
    sh, hs = agg_shard
    cases = [
        [("term", 0, ">", 100.5)],
        [("term", 0, "<", 100.25)],
        [("term", 1, ">=", 0)],
        [("term", 1, "<", 100.5)],                       # int column against a float constant (Int64ToFloat64Slice)
        [("term", 2, "=", 1)],
        [("term", 3, ">", 1000.0), ("term", 5, "!=", 1), "and"],
        [("term", 0, ">", 100.9), ("term", 4, "<", -2000), "or"],
        [("term", 0, ">", 100.2), ("term", 0, "<=", 100.8), "and", ("term", 2, "=", 0), "or"],
        [("term", 0, ">", 200.0)],                       # nothing survives
    ]
    for flt in cases:
        run_both(sh, hs.desc, [("count", 1), ("sum", 1), ("sum", 0), ("count", 2)], 60 * SEC, T0, T0 + 4320 * SEC, f"where {flt}", filter=flt)
        run_both(sh, hs.desc, [("max", 3)], 300 * SEC, T0 + 100 * SEC, T0 + 4000 * SEC, f"where {flt} max", filter=flt)
        run_both(sh, hs.desc, [("first", 4)], 3600 * SEC, T0, T0 + 4320 * SEC, f"where {flt} first", filter=flt, group="series")


def test_nan_and_tie_semantics():
    """NaN handling (strict compares, sticky first NaN of a record window) and tie-breaks must follow the reducers exactly.
    NaN can only reach a page through the raw/Snappy routes (FloatArrayEncodeAll rejects it), so the shard is built from
    4-row segments (n <= 4 -> floatCompressedNull, float.go:26,96): windows then span many records, which is exactly where
    the record-boundary-dependent NaN behaviour of the reducers shows."""
    n, nsegs, nser = 4, 40, 6
    rng = np.random.default_rng(21)
    series = []
    for s in range(nser):
        v = np.round(rng.random(n * nsegs) * 4) / 4  # many ties
        v[rng.integers(0, n * nsegs, 25)] = np.nan
        if s == 1:
            v[0] = np.nan      # window that starts with NaN
            v[8] = np.nan      # a record that starts with NaN inside a window spanning several records
        series.append(v)
    pages, tpages, tmins, tmaxs = [], [], [], []
    for s in range(nser):
        for g in range(nsegs):
            pages.append(oracle.field_page_encode(L.TYPE_FLOAT, series[s][g * n:(g + 1) * n]))
            t = T0 + (np.arange(n, dtype=np.int64) + g * n) * SEC
            tpages.append(oracle.time_page_encode(t)); tmins.append(t[0]); tmaxs.append(t[-1])
    blob, offs, lens = [], [], []
    pos = 0
    for p in pages + tpages:
        offs.append(pos); lens.append(p.size); blob.append(p); pos += p.size
    data = np.concatenate(blob)
    nseg = nser * nsegs
    sh = Shard.open(data, np.arange(1, nser + 1), np.arange(0, nseg + 1, nsegs), tmins, tmaxs,
                    [("v", L.TYPE_FLOAT, offs[:nseg], lens[:nseg])], offs[nseg:], lens[nseg:])
    ex = sh.export()
    sd = oracle.shard_desc_from_export(ex)
    tmax = T0 + n * nsegs * SEC
    for flags in (0, L.Q_NO_FUSED):
        for iv in (7 * SEC, 60 * SEC, 0):
            for f in ALL6:
                run_both(sh, sd, [(f, 0)], iv, T0, tmax, f"nan {f} iv={iv}", flags=flags, folded=False)
            run_both(sh, sd, [(f, 0) for f in ALL6], iv, T0, tmax, "nan multi", flags=flags, folded=False)
            run_both(sh, sd, [("max", 0)], iv, T0, tmax, "nan max per series", flags=flags, group="series")
            run_both(sh, sd, [("min", 0)], iv, T0 + 3 * SEC, tmax - 5 * SEC, "nan min mid-range", flags=flags, folded=False)
            run_both(sh, sd, [("count", 0)], iv, T0, tmax, "nan count folded", flags=flags)
    sh.close()


def test_records_next_matches_dense(agg_shard):
    sh, hs = agg_shard
    q = AggQuery(sh, [("sum", 3), ("count", 3), ("last", 3)], 60 * SEC, T0, T0 + 4320 * SEC, group="series", chunk_size=16).run()
    d = q.dense_host()
    nb = d["n_buckets"]
    seen = 0
    for rec in q.records():
        g = rec["group"]
        assert rec["sid"] == g + 1
        assert rec["rows"] <= 16
        b = (rec["times"] - d["start"]) // (60 * SEC)
        for k in range(3):
            col = rec["cols"][k]
            cells = g * nb + b
            assert np.array_equal(col["valid"], d["cols"][k]["valid"][cells].astype(bool))
            want = d["cols"][k]["values"][cells][col["valid"]]
            assert np.array_equal(col["values"].view(np.uint64), want.view(np.uint64))
        assert rec["cols"][2]["times"] is not None  # RecMeta.Times for last() in a multi-call query
        seen += rec["rows"]
    any_valid = np.zeros(d["n_groups"] * nb, bool)
    for k in range(3):
        any_valid |= d["cols"][k]["valid"].astype(bool)
    assert seen == int(any_valid.sum())
    q.close()


def test_larger_shard_properties():
    """Size-independent checks on a shard the oracle would take long on: counts add up, sums are linear,
    fused == generic bitwise, per-series folds to all-series."""
    n_series, rows = 300, 20_000
    sh = Shard.synth(n_series, rows, [(L.TYPE_FLOAT, L.SYNTH_F_HI, 0)], t0=T0, dt=SEC, seed=5)
    info = sh.info()
    assert info["n_rows"] == n_series * rows and info["n_segments"] == n_series * 20
    tmax = T0 + (rows - 1) * SEC
    qa = AggQuery(sh, [("sum", 0), ("count", 0), ("max", 0), ("min", 0)], 60 * SEC, T0, tmax, flags=L.Q_STRICT_ORDER).run()
    qb = AggQuery(sh, [("sum", 0), ("count", 0), ("max", 0), ("min", 0)], 60 * SEC, T0, tmax, flags=L.Q_NO_FUSED).run()
    qf = AggQuery(sh, [("sum", 0), ("count", 0), ("max", 0), ("min", 0)], 60 * SEC, T0, tmax).run()  # folded order
    assert qa.stats()["path"] == 2 and qf.stats()["path"] == 3 and qf.stats()["per_series_cells_used"] == 0 and qf.stats()["il_state"] == 1
    f = qf.dense_host()
    a, b = qa.dense_host(), qb.dense_host()
    for k in range(4):
        assert np.array_equal(a["cols"][k]["valid"], b["cols"][k]["valid"])
        assert np.array_equal(_bits(a["cols"][k]["values"]), _bits(b["cols"][k]["values"]))
    for k in (1, 2, 3):  # count, max, min: the folded order changes nothing
        assert np.array_equal(a["cols"][k]["valid"], f["cols"][k]["valid"]) and np.array_equal(_bits(a["cols"][k]["values"]), _bits(f["cols"][k]["values"]))
    assert np.allclose(a["cols"][0]["values"], f["cols"][0]["values"], rtol=SUM_RTOL, atol=0)
    cnt = a["cols"][1]["values"]
    assert int(cnt.sum()) == n_series * rows
    assert np.all(a["cols"][2]["values"][a["cols"][2]["valid"] > 0] < 101.0) and np.all(a["cols"][3]["values"][a["cols"][3]["valid"] > 0] >= 100.0)
    mean = a["cols"][0]["values"] / np.maximum(cnt, 1)
    assert np.all(np.abs(mean[cnt > 0] - 100.5) < 0.05)
    qs = AggQuery(sh, [("sum", 0), ("count", 0)], 60 * SEC, T0, tmax, group="series").run()
    s = qs.dense_host()
    per = s["cols"][0]["values"].reshape(n_series, -1)
    # folding the per-series sums in series order reproduces the all-series sums bitwise
    acc = np.zeros(per.shape[1])
    for i in range(n_series):
        acc = per[i] + acc
    assert np.array_equal(acc.view(np.uint64), a["cols"][0]["values"].view(np.uint64))
    assert np.array_equal(s["cols"][1]["values"].reshape(n_series, -1).sum(0), cnt)
    for q in (qa, qb, qs, qf):
        q.close()
    sh.close()


def test_encode_pages_roundtrip_on_device():
    """og_encode_pages (K7) output decodes back to the input through og_shard_open + og_decode_segment."""
    import torch
    rng = np.random.default_rng(8)
    nseg, rps = 6, 1000
    vals = np.cumsum(rng.integers(-3, 4, nseg * rps)).astype(np.float64)
    dv = torch.from_numpy(vals).cuda()
    out = torch.zeros(nseg * 8704, dtype=torch.uint8, device="cuda")
    off = torch.zeros(nseg, dtype=torch.int64, device="cuda")
    ln = torch.zeros(nseg, dtype=torch.int32, device="cuda")
    total = C.c_uint64()
    L.check(L.lib().og_encode_pages(L.TYPE_FLOAT, 0, dv.data_ptr(), None, None, nseg, rps, out.data_ptr(), out.numel(),
                                    off.data_ptr(), ln.data_ptr(), C.byref(total)), "og_encode_pages")
    pages = out.cpu().numpy()
    offs, lens = off.cpu().numpy(), ln.cpu().numpy()
    assert int(lens.sum()) == total.value
    for g in range(nseg):
        want = oracle.field_page_encode(L.TYPE_FLOAT, vals[g * rps:(g + 1) * rps])
        got = pages[offs[g]:offs[g] + lens[g]]
        assert np.array_equal(got, want), f"segment {g}"


def _ragged_shard(seg_counts, n=500):
    """Series with different numbers of segments (so lane groups are 32 consecutive segments, not 32 series)."""
    rng = np.random.default_rng(12)
    pages, tpages, tmins, tmaxs, ssb = [], [], [], [], [0]
    for k in seg_counts:
        for g in range(k):
            v = 100.0 + rng.random(n)
            if g == 1:
                v = rng.integers(0, 2**62, n).astype(np.uint64).view(np.float64)  # incompressible -> raw page
                v = np.where(np.isfinite(v), v, 1.0)
            pages.append(oracle.field_page_encode(L.TYPE_FLOAT, v))
            t = T0 + (np.arange(n, dtype=np.int64) + g * n) * SEC
            tpages.append(oracle.time_page_encode(t)); tmins.append(t[0]); tmaxs.append(t[-1])
        ssb.append(ssb[-1] + k)
    blob, offs, lens, pos = [], [], [], 0
    for p in pages + tpages:
        offs.append(pos); lens.append(p.size); blob.append(p); pos += p.size
    nseg = ssb[-1]
    sh = Shard.open(np.concatenate(blob), np.arange(1, len(seg_counts) + 1), ssb, tmins, tmaxs,
                    [("v", L.TYPE_FLOAT, offs[:nseg], lens[:nseg])], offs[nseg:], lens[nseg:])
    return sh, oracle.shard_desc_from_export(sh.export()), T0 + max(seg_counts) * n * SEC


@pytest.mark.gpu
def test_ragged_series_use_consecutive_segment_groups():
    sh, sd, tmax = _ragged_shard([1, 2, 3, 5, 8, 13, 2, 1, 40])
    for calls in ([("sum", 0), ("count", 0), ("max", 0)], [("min", 0)], [("first", 0), ("last", 0)]):
        for group in ("all", "series"):
            run_both(sh, sd, calls, 60 * SEC, T0, tmax, f"ragged {calls} {group}", group=group)
    run_both(sh, sd, [("sum", 0), ("max", 0)], 45 * SEC, T0 + 123 * SEC, T0 + 2345 * SEC, "ragged mid-range")
    sh.close()


@pytest.mark.gpu
@pytest.mark.parametrize("chunk", ["32", "7"])
def test_multi_chunk_plans(monkeypatch, chunk):
    """OGPU_CHUNK_SERIES forces several chunks of series per query (as happens when the cell matrix outgrows memory)."""
    monkeypatch.setenv("OGPU_CHUNK_SERIES", chunk)
    cols = [(L.TYPE_FLOAT, L.SYNTH_F_HI, 0), (L.TYPE_INT, L.SYNTH_INT_WALK, 30)]
    sh = Shard.synth(100, 3000, cols, t0=T0, dt=SEC, seed=5)
    hs = oracle.HostShard(100, 3000, cols, t0=T0, dt=SEC, seed=5)
    tmax = T0 + 2999 * SEC
    run_both(sh, hs.desc, [("sum", 0), ("count", 0), ("max", 0)], 60 * SEC, T0, tmax, "chunks fast")
    run_both(sh, hs.desc, [("min", 0)], 300 * SEC, T0, tmax, "chunks fast selector", group="series")
    run_both(sh, hs.desc, [("sum", 1), ("last", 1)], 60 * SEC, T0, tmax, "chunks general int")
    run_both(sh, hs.desc, [("count", 1), ("sum", 0)], 60 * SEC, T0, tmax, "chunks tile", filter=[("term", 0, ">", 100.5)])
    run_both(sh, hs.desc, [("max", 0), ("count", 1)], 120 * SEC, T0, tmax, "chunks map", group="map", series_group=np.arange(100) % 3, n_groups=3)
    sh.close()
    ragged, sd, tm = _ragged_shard([3, 1, 4, 1, 5, 9, 2, 6])
    run_both(ragged, sd, [("sum", 0), ("count", 0), ("max", 0)], 60 * SEC, T0, tm, "chunks ragged")
    ragged.close()


def _shard_from_series(series_values, n=1000):
    """Regular shard: every series has len(values)/n segments of n rows, 1 s cadence."""
    pages, tpages, tmins, tmaxs, ssb = [], [], [], [], [0]
    for v in series_values:
        k = len(v) // n
        for g in range(k):
            pages.append(oracle.field_page_encode(L.TYPE_FLOAT, v[g * n:(g + 1) * n]))
            t = T0 + (np.arange(n, dtype=np.int64) + g * n) * SEC
            tpages.append(oracle.time_page_encode(t)); tmins.append(t[0]); tmaxs.append(t[-1])
        ssb.append(ssb[-1] + k)
    blob, offs, lens, pos = [], [], [], 0
    for p in pages + tpages:
        offs.append(pos); lens.append(p.size); blob.append(p); pos += p.size
    nseg = ssb[-1]
    sh = Shard.open(np.concatenate(blob), np.arange(1, len(series_values) + 1), ssb, tmins, tmaxs,
                    [("v", L.TYPE_FLOAT, offs[:nseg], lens[:nseg])], offs[nseg:], lens[nseg:])
    return sh, oracle.shard_desc_from_export(sh.export())


def test_lanes_out_of_step():
    """Series of very different entropy in one binning domain: the lanes of a group drift apart by hundreds of ring rows, so
    the heavy ones sit rounds out (shared-window residency rule) and close their windows at different moments than the others
    (per-bucket accumulators of the folding warp).  Results must not change."""
    rng = np.random.default_rng(77)
    n_series, rows = 40, 3000
    series = []
    for s in range(n_series):
        k = 4 + (s * 48) // n_series  # 4 .. 51 random mantissa bits below the binary point
        series.append(100.0 + np.floor(rng.random(rows) * 2.0**k) / 2.0**k)
    sh, sd = _shard_from_series(series)
    tmax = T0 + (rows - 1) * SEC
    for calls in ([("sum", 0), ("count", 0), ("max", 0)], [("min", 0)], [("first", 0), ("last", 0), ("sum", 0)]):
        run_both(sh, sd, calls, 60 * SEC, T0, tmax, f"out of step {calls}")
    run_both(sh, sd, [("sum", 0), ("max", 0)], 45 * SEC, T0 + 777 * SEC, T0 + 2500 * SEC, "out of step mid-range")
    run_both(sh, sd, [("max", 0)], 60 * SEC, T0, tmax, "out of step per series", group="series")
    q = AggQuery(sh, [("sum", 0), ("count", 0)], 60 * SEC, T0, tmax).run()
    st = q.stats()
    assert st["path"] == 3 and st["per_series_cells_used"] == 0, st  # drifting lanes stay on the folded path (shared-memory window accumulators)
    q.close()
    sh.close()


def test_folded_path_selectors_and_ties():
    """One tagset, folded order: selector tie-breaks across series (equal extremes -> earlier time; equal times -> larger
    value for first/last) must survive the butterfly fold.  Values are drawn from a tiny set so ties are everywhere."""
    rng = np.random.default_rng(5)
    n_series, rows = 70, 2000
    series = [100.0 + rng.integers(0, 4, rows) * 0.0625 + (rng.random(rows) < 0.02) * rng.random(rows) for _ in range(n_series)]
    sh, sd = _shard_from_series(series)
    tmax = T0 + (rows - 1) * SEC
    for iv in (60 * SEC, 7 * SEC, 1000 * SEC, 0):
        for f in ALL6:
            run_both(sh, sd, [(f, 0)], iv, T0, tmax, f"ties {f} iv={iv}")
        run_both(sh, sd, [(f, 0) for f in ALL6], iv, T0, tmax, f"ties multi iv={iv}")
    run_both(sh, sd, [("max", 0), ("count", 0)], 60 * SEC, T0 + 500 * SEC + 3, T0 + 1500 * SEC, "ties mid-range")
    sh.close()


def test_two_stage_merge_of_per_series_cells(monkeypatch):
    """One tagset, order not pinned, per-series cells (multi-column / WHERE queries, general codecs): the cells are folded by
    blocks of series in parallel and the block partials by k_merge_folded.  OGPU_FORCE_BLOCKMERGE enables it below its size
    threshold.  Everything but float sums is bitwise; float sums within 1e-12."""
    monkeypatch.setenv("OGPU_FORCE_BLOCKMERGE", "1")
    cols = [(L.TYPE_FLOAT, L.SYNTH_F_HI, 30), (L.TYPE_INT, L.SYNTH_INT_WALK, 0), (L.TYPE_BOOL, L.SYNTH_BOOL, 100)]
    n_series, rows = 700, 3000
    sh = Shard.synth(n_series, rows, cols, t0=T0, dt=SEC, seed=9)
    hs = oracle.HostShard(n_series, rows, cols, t0=T0, dt=SEC, seed=9, threads=4)
    tmax = T0 + (rows - 1) * SEC
    cases = [([("count", 1), ("sum", 1), ("sum", 0), ("count", 2)], [("term", 0, ">", 100.5)]),
             ([(f, 0) for f in ALL6], None), ([("max", 1)], [("term", 2, "=", 1)]), ([("first", 0)], None), ([("last", 1), ("min", 0)], None)]
    for calls, flt in cases:
        q = AggQuery(sh, calls, 60 * SEC, T0, tmax, filter=flt).run()
        ref = oracle.scan(hs.desc, q.desc, threads=1)
        compare_dense(q.dense_host(), ref, calls, len(calls) > 1, f"blockmerge {calls}", float_sum_exact=False)
        q.close()
    sh.close()


def test_column_at_a_time_kernel_and_pull_iterator_kernel_agree_with_the_oracle(agg_shard, monkeypatch):
    """Queries over several columns / one WHERE term run k_fused_cols (path 5) on const-delta shards; OGPU_NO_COLS selects the
    older k_fused_multi (path 4).  Both must equal the oracle bitwise (run_both) on: columns with and without nulls, every
    call kind, ranges that cut segments, windows shorter than the cadence, one window for everything."""
    sh, hs = agg_shard
    tmax = T0 + 4320 * SEC
    cases = [
        ([("sum", 0), ("count", 4), ("max", 3), ("last", 5), ("min", 1)], None, 60 * SEC, T0, tmax, {}),
        ([("count", 1), ("sum", 1), ("sum", 3), ("count", 5)], [("term", 3, ">", 1000.0)], 60 * SEC, T0, tmax, {}),
        ([("count", 1), ("sum", 0), ("count", 2), ("sum", 4)], [("term", 4, "<", 0)], 7 * SEC, T0 + 1234 * SEC + 5, T0 + 3456 * SEC + 7, {}),
        ([("first", 0), ("last", 0), ("min", 3), ("max", 3)], [("term", 2, "=", 1)], 3600 * SEC, T0 - 500 * SEC, T0 + 10_000 * SEC, dict(offset=7 * SEC)),
        ([("sum", 3), ("count", 3), ("sum", 4), ("count", 4), ("count", 5)], None, 0, T0 + 999 * SEC, T0 + 1001 * SEC, {}),
        ([("max", 4)], [("term", 0, ">", 100.5)], 61 * SEC, T0 + 17, T0 + 4000 * SEC, dict(offset=-13 * SEC, group="series")),
        ([("sum", 1), ("sum", 0)], [("term", 5, "!=", 1)], 300 * SEC, T0, tmax, dict(group="map", series_group=[2, 0, 1, 0, 2, 2, 0], n_groups=3)),
    ]
    for no_cols, want in (("", 5), ("1", 4)):
        if no_cols:
            monkeypatch.setenv("OGPU_NO_COLS", no_cols)
        for calls, flt, iv, t0, t1, kw in cases:
            q = AggQuery(sh, calls, iv, t0, t1, filter=flt, **kw).run()
            ncols = len({c for _, c in calls} | {t[1] for t in (flt or []) if isinstance(t, tuple)})
            assert q.stats()["path"] == (want if want == 5 or ncols <= 4 else 0), (calls, flt)  # the pull-iterator kernel takes <= 4 columns
            q.close()
            run_both(sh, hs.desc, calls, iv, t0, t1, f"cols={want} {calls} where {flt}", filter=flt, **kw)
    monkeypatch.delenv("OGPU_NO_COLS")
    # cadence longer than the window (windows without rows), and all rows on one timestamp is not a const-delta page the encoder
    # produces; long segments (> 1024 rows) fall back to the pull-iterator kernel
    cols = [(L.TYPE_FLOAT, L.SYNTH_F_LO, 0), (L.TYPE_INT, L.SYNTH_INT_WALK, 300), (L.TYPE_BOOL, L.SYNTH_BOOL, 0)]
    hs2 = oracle.HostShard(5, 2345, cols, t0=T0, dt=90 * SEC, seed=77)
    sh2 = Shard.open_desc(hs2.desc, keepalive=hs2)
    for flt in (None, [("term", 0, ">", 1000.0)]):
        run_both(sh2, hs2.desc, [("sum", 0), ("count", 1), ("count", 2), ("sum", 1)], 60 * SEC, T0 + 100 * SEC, T0 + 2000 * 90 * SEC, f"sparse windows where {flt}", filter=flt)
    sh2.close()
    hs3 = oracle.HostShard(3, 5000, cols, t0=T0, dt=SEC, seed=78, rows_per_segment=2000)
    sh3 = Shard.open_desc(hs3.desc, keepalive=hs3)
    q = AggQuery(sh3, [("sum", 0), ("count", 1)], 60 * SEC, T0, T0 + 4999 * SEC).run()
    assert q.stats()["path"] == 4
    q.close()
    run_both(sh3, hs3.desc, [("sum", 0), ("count", 1)], 60 * SEC, T0, T0 + 4999 * SEC, "2000-row segments")
    sh3.close()
