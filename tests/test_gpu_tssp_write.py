"""og_shard_write_tssp on the device against tests/tssp_write_model.py (the Python restatement of the reference's writer):
the file byte for byte, every column CRC against zlib, the file reopened through og_tssp_parse and queried against its source,
pre-aggregation cells against the oracle's aggregates, merged and downsampled shards, and every refusal."""
import struct
import zlib

import numpy as np
import pytest

import oracle
import tssp_write_model as M
from opengemini_b200 import AggQuery, Shard, write_tssp
from opengemini_b200 import _lib as L

pytestmark = pytest.mark.gpu
T0, SEC = 1_700_000_000_000_000_000, 1_000_000_000


@pytest.fixture(autouse=True)
def _device():
    Shard.init(0)


# ---------------------------------------------------------------- shards built row by row, so the model never reads a page
def _string_page(valid):
    rows, nil = len(valid), int(len(valid) - valid.sum())
    payload = b"\x10opaque-string-block"
    if nil == 0:
        return bytes([34]) + struct.pack(">I", rows) + payload
    if nil == rows:
        return bytes([44]) + struct.pack(">I", rows)
    bm = np.packbits(valid.astype(np.uint8), bitorder="little").tobytes()
    return bytes([L.TYPE_STRING]) + struct.pack(">I", len(bm)) + bm + struct.pack(">II", 0, nil) + payload


def _cells(kind, rng, n):
    if kind == "f_hi":
        return 100 + rng.random(n)                                     # Gorilla, high entropy
    if kind == "f_lo":
        return np.repeat(20 + np.cumsum(rng.integers(-2, 3, (n + 3) // 4)) / 3.0, 4)[:n]   # Gorilla, mostly repeated values
    if kind == "f_raw":
        return rng.standard_normal(n) * 10.0 ** rng.integers(-300, 300, n)
    if kind == "f_rle":
        return np.repeat(rng.choice([1.5, 0.0, -7.25], 4), (n + 3) // 4)[:n]     # at most four runs: more than eight would be Snappy
    if kind == "f_same":
        return np.full(n, 4.5)
    if kind == "f_edge":                                               # NaN, infinities, +-MaxFloat64, signed zeros: raw pages of <= 4 rows
        return rng.choice([np.nan, np.inf, -np.inf, M.MAX_F64, -M.MAX_F64, 0.0, -0.0, 1.0], n)
    if kind == "i_const":
        return (7 + 3 * np.arange(n)).astype(np.int64)
    if kind == "i_s8b":
        return np.cumsum(rng.integers(-1000, 1001, n)).astype(np.int64)
    if kind == "i_wide":                                              # one value per Simple8b word; raw pages below three rows
        return rng.integers(-(1 << 57), 1 << 57, n).astype(np.int64)
    if kind == "bool":
        return rng.integers(0, 2, n).astype(np.uint8)
    if kind == "str":
        return np.zeros(n, np.uint8)
    raise KeyError(kind)


_TYPE = dict(f=L.TYPE_FLOAT, i=L.TYPE_INT, b=L.TYPE_BOOL, s=L.TYPE_STRING)


def make_chunks(seed, n_series, columns, seg_rows, time_kinds=("const",), sid0=1, t0=T0):
    """columns: [(name, kind, null share)] sorted by name; seg_rows(rng, series) -> rows of each segment of the series."""
    rng = np.random.default_rng(seed)
    chunks = []
    for s in range(n_series):
        times, t = [], t0 + int(rng.integers(0, 50)) * SEC
        for k, n in enumerate(seg_rows(rng, s)):
            kind = time_kinds[(s + k) % len(time_kinds)]
            if kind == "const":
                tt = t + np.arange(n, dtype=np.int64) * SEC
            else:                                                       # irregular: Simple8b; two-row segments give raw time pages
                tt = t + np.cumsum(rng.integers(1, 90, n)).astype(np.int64) * SEC
            times.append(tt.astype(np.int64))
            t = int(tt[-1]) + SEC
        cols = []
        for name, kind, nulls in columns:
            typ = _TYPE[kind[0]]
            pages, rows = [], []
            for tt in times:
                n = tt.size
                cells = _cells(kind, rng, n)
                valid = np.ones(n, bool) if nulls == 0 else np.zeros(n, bool) if nulls >= 1 else rng.random(n) >= nulls
                page = _string_page(valid) if typ == L.TYPE_STRING else oracle.field_page_encode(typ, cells, valid.astype(np.uint8)).tobytes()
                pages.append(page)
                rows.append((cells.tolist(), valid.tolist()))
            cols.append((name.encode(), typ, pages, rows))
        chunks.append(dict(sid=sid0 + 3 * s, tmin=[int(t[0]) for t in times], tmax=[int(t[-1]) for t in times], times=[t.tolist() for t in times],
                           time_pages=[oracle.time_page_encode(t).tobytes() for t in times], columns=cols))
    return chunks


def shard_desc(chunks, seed=0):
    """An L.ShardDesc whose data holds the pages in shuffled order with gaps between them: nothing like the file's layout."""
    rng = np.random.default_rng(seed)
    names = [(n.decode(), ty) for n, ty, _p, _r in chunks[0]["columns"]]
    nseg = sum(len(c["time_pages"]) for c in chunks)
    pages = []                                   # (column index or -1 for time, global segment, bytes)
    ssb, g = [0], 0
    for c in chunks:
        assert [(n.decode(), ty) for n, ty, _p, _r in c["columns"]] == names
        for k in range(len(c["time_pages"])):
            pages.append((-1, g + k, c["time_pages"][k]))
            for ci, (_n, _ty, pg, _r) in enumerate(c["columns"]):
                pages.append((ci, g + k, pg[k]))
        g += len(c["time_pages"])
        ssb.append(g)
    po = np.zeros((len(names) + 1, nseg), np.uint64)
    pl = np.zeros((len(names) + 1, nseg), np.uint32)
    blob = bytearray(b"\xee" * 5)
    for i in rng.permutation(len(pages)):
        ci, seg, b = pages[i]
        po[ci, seg], pl[ci, seg] = len(blob), len(b)
        blob += b + b"\xdd" * int(rng.integers(0, 4))
    d = Shard.desc(bytes(blob), [c["sid"] for c in chunks], ssb, [t for c in chunks for t in c["tmin"]], [t for c in chunks for t in c["tmax"]],
                   [(n, ty, po[i], pl[i]) for i, (n, ty) in enumerate(names)], po[-1], pl[-1])
    return d


MIXED = [("a_fhi", "f_hi", 0), ("b_flo", "f_lo", 0.05), ("c_fraw", "f_raw", 0), ("d_frle", "f_rle", 0), ("e_fsame", "f_same", 0.05),
         ("f_null", "f_hi", 1), ("g_iconst", "i_const", 0), ("h_is8b", "i_s8b", 0.05), ("i_iwide", "i_wide", 0), ("j_bool", "bool", 0),
         ("k_booln", "bool", 0.4), ("l_str", "str", 0.05), ("m_inull", "i_s8b", 1)]


def _mixed_rows(rng, s):
    if s == 0:
        return [1]                               # a series with a single row
    return [int(x) for x in rng.choice([1, 2, 5, 120, 1000], int(rng.integers(1, 5)))]


SHARDS = {
    "mixed": lambda: make_chunks(11, 9, MIXED, _mixed_rows, ("const", "s8b")),
    "edge_floats": lambda: make_chunks(12, 40, [("x", "f_edge", 0), ("y", "f_edge", 0.3)], lambda rng, s: [int(x) for x in rng.integers(1, 5, int(rng.integers(1, 4)))]),
    "meta_blocks": lambda: make_chunks(13, 1100, [("v", "i_const", 0)], lambda rng, s: [3]),
    "long_chunk": lambda: make_chunks(14, 2, [("v", "f_hi", 0.05), ("w", "bool", 0.5)], lambda rng, s: [int(x) for x in rng.integers(1, 4, 3000)]),
}


def _check_crcs(f):
    p = M.parse(f)
    for ch in p["chunks"]:
        for c in ch["columns"]:
            assert c["crc"] == zlib.crc32(b"".join(f[o:o + z] for o, z in c["segs"])), (ch["sid"], c["name"])
    return p


# ---------------------------------------------------------------- 1, 2: the file equals the model's; CRCs
@pytest.mark.parametrize("name", list(SHARDS))
def test_file_equals_the_model_byte_for_byte(name):
    chunks = SHARDS[name]()
    d = shard_desc(chunks, seed=1)
    sh = Shard.open_desc(d)
    try:
        timing = {}
        got = write_tssp(sh, "m_" + name, timing=timing)
        want = M.build(chunks, ("m_" + name).encode())
        assert len(got) == len(want)
        assert got == want
        assert set(timing) == {"preagg", "layout_gather_crc", "metadata_d2h", "host_assembly"} and all(v >= 0 for v in timing.values())
        p = _check_crcs(got)
        if name == "meta_blocks":
            assert [m["count"] for m in p["meta_index"]] == [512, 512, 76]
        if name == "long_chunk":
            assert len(p["chunks"][0]["tmin"]) == 3000 and min(z for _o, z in p["chunks"][0]["columns"][1]["segs"]) <= 2
    finally:
        sh.close()


def test_series_sub_range():
    chunks = SHARDS["mixed"]()
    sh = Shard.open_desc(shard_desc(chunks, seed=2))
    try:
        assert write_tssp(sh, "part", series=(2, 6)) == M.build(chunks[2:6], b"part")
        assert write_tssp(sh, "part", series=(8, 9)) == M.build(chunks[8:9], b"part")
        assert write_tssp(sh, "part", series=(0, 9)) == write_tssp(sh, "part")
    finally:
        sh.close()


# ---------------------------------------------------------------- 3: reopen and compare with the source
def _dense(sh, calls, interval, tmin, tmax, **kw):
    q = AggQuery(sh, calls, interval, tmin, tmax, flags=L.Q_STRICT_ORDER, **kw)
    try:
        return q.run().dense_host()
    finally:
        q.close()


def _same_answers(a, b, col_types, filter_col=None):
    ia, ib = a.info(), b.info()
    assert ia == ib
    tmin, tmax = ia["tmin"], ia["tmax"]
    span = max(1, (tmax - tmin) // 7)
    n = 0
    for c, ty in enumerate(col_types):
        funcs = {L.TYPE_STRING: ["count"], L.TYPE_BOOL: ["count", "min", "max", "first", "last"]}.get(ty, ["count", "sum", "min", "max", "first", "last"])
        for calls in ([(f, c) for f in funcs[:3]], [(f, c) for f in funcs[3:]] or None):
            if not calls:
                continue
            variants = [dict(), dict(group="series")]
            if filter_col is not None and ty != L.TYPE_STRING:
                variants.append(dict(filter=[("term", filter_col, ">", 0)]))
            for interval in (0, span):
                for kw in variants:
                    x, y = _dense(a, calls, interval, tmin, tmax, **kw), _dense(b, calls, interval, tmin, tmax, **kw)
                    for cx, cy in zip(x["cols"], y["cols"]):
                        assert np.array_equal(cx["valid"], cy["valid"])
                        m = cx["valid"].astype(bool)
                        assert np.array_equal(cx["values"].view(np.uint64)[m], cy["values"].view(np.uint64)[m]), (c, calls, interval, kw)
                        if cx["times"] is not None:
                            assert np.array_equal(cx["times"][m], cy["times"][m])
                    n += 1
    return n


def _referenced_pages(ex):
    return [[ex["data"][int(o):int(o) + int(z)].tobytes() for o, z in zip(ex["page_off"][c], ex["page_len"][c])] for c in range(ex["page_off"].shape[0])]


@pytest.mark.parametrize("name", ["mixed", "long_chunk"])
def test_written_file_reopens_as_the_same_shard(name):
    chunks = SHARDS[name]()
    src = Shard.open_desc(shard_desc(chunks, seed=3))
    back = Shard.open_tssp(write_tssp(src, "rt"))
    try:
        assert back.measurement == "rt"
        ea, eb = src.export(), back.export()
        for k in ("sids", "series_seg_begin", "seg_tmin", "seg_tmax", "col_types"):
            assert np.array_equal(ea[k], eb[k]), k
        assert _referenced_pages(ea) == _referenced_pages(eb)
        types = [ty for _n, ty, _p, _r in chunks[0]["columns"]]
        assert _same_answers(src, back, types, filter_col=7 if name == "mixed" else None) >= 16
    finally:
        src.close()
        back.close()


# ---------------------------------------------------------------- 4: pre-aggregation cells against the oracle's aggregates
def test_preagg_cells_equal_the_oracle_per_series_aggregates():
    """Where the builders' rule and the query reducers' rule coincide: columns without NaN or +-MaxFloat64, more than one value
    (the six-field form); the times of min / max where no value repeats across segments.  A float sum coincides only for a chunk of
    one segment (series 0 here): the reducers add per-segment sums, the builder adds row by row across segments.  That sum, bool
    times and the NaN cases are pinned by the model in the byte-for-byte tests."""
    cols = [("a_fhi", "f_hi", 0), ("b_flo", "f_lo", 0.05), ("c_frle", "f_rle", 0), ("d_is8b", "i_s8b", 0.05), ("e_iwide", "i_wide", 0)]
    chunks = make_chunks(21, 6, cols, lambda rng, s: [900] if s == 0 else [1000, 1000, int(rng.integers(2, 900))], ("const", "s8b"))
    d = shard_desc(chunks, seed=4)
    sh = Shard.open_desc(d)
    try:
        p = M.parse(write_tssp(sh, "agg"))
        info = sh.info()
        for c, (_n, kind, _nulls) in enumerate(cols):
            def ref_of(funcs):
                q = AggQuery(sh, [(f, c) for f in funcs], 0, info["tmin"], info["tmax"], group="series", flags=L.Q_STRICT_ORDER)
                try:
                    return oracle.scan(d, q.desc, threads=1)
                finally:
                    q.close()
            ref = ref_of(("min", "max", "sum", "count"))
            tmin_ref, tmax_ref = ref_of(("min",)), ref_of(("max",))   # a single call carries the time of the selected row
            is_f = kind[0] == "f"
            for s, ch in enumerate(p["chunks"]):
                r = M._R(ch["columns"][c]["preagg"])
                assert len(r.b) == 48
                val = (lambda: r.u64()) if is_f else (lambda: r.i64() & M.M64)
                got = dict(min=val(), max=val(), mint=r.i64(), maxt=r.i64(), sum=val(), count=r.i64())
                want = {k: int(ref["cols"][i]["values"][s]) for i, k in enumerate(("min", "max", "sum", "count")) if not (k == "sum" and is_f and s > 0)}
                assert {k: got[k] for k in want} == want, (c, s)
                if s == 0 or kind in ("f_hi", "i_wide"):   # equal values in different segments: the reducers' tie rule is not the builder's
                    assert (got["mint"], got["maxt"]) == (int(tmin_ref["cols"][0]["times"][s]), int(tmax_ref["cols"][0]["times"][s])), (c, s)
    finally:
        sh.close()


# ---------------------------------------------------------------- 5: merged and downsampled shards
def test_merged_shard_writes_its_live_pages():
    cols = [("u", "f_hi", 0), ("v", "i_s8b", 0.05)]
    ordered = make_chunks(31, 5, cols, lambda rng, s: [1000, 1000, 400], t0=T0)
    late = make_chunks(32, 5, cols, lambda rng, s: [300], ("s8b",), t0=T0 + 500 * SEC)   # rows inside the first ordered segments
    merged = Shard.open_files([(M.build(ordered, b"m"), False), (M.build(late, b"m"), True)])
    ordered_only = Shard.open_files([(M.build(ordered, b"m"), False)])
    back = None
    try:
        # without a merge the shard keeps the file's region, CRCs and metadata included: the writer takes only the pages from it
        eo = ordered_only.export()
        referenced_o = int(eo["page_len"].sum())
        assert referenced_o < eo["data"].size
        assert M.parse(write_tssp(ordered_only, "m"))["trailer"]["data_size"] == referenced_o + 4 * 3 * 5
        mi = merged.merge_info()
        assert mi["series_merged"] == 5 and mi["segments_rewritten_in"] > 0
        f = write_tssp(merged, "m")
        _check_crcs(f)
        ex = merged.export()
        referenced = int(ex["page_len"].sum())
        assert referenced == ex["data"].size, "the merged shard holds only the pages its directory references"
        p = M.parse(f)
        assert p["trailer"]["data_size"] == referenced + 4 * 3 * 5        # only referenced pages, plus one CRC per column of a chunk
        back = Shard.open_tssp(f)
        assert _referenced_pages(ex) == _referenced_pages(back.export())
        assert _same_answers(merged, back, [L.TYPE_FLOAT, L.TYPE_INT], filter_col=1) > 10
        # the count cells are those of the merged rows
        info = merged.info()
        x = _dense(merged, [("count", 1)], 0, info["tmin"], info["tmax"], group="series")
        for s, ch in enumerate(p["chunks"]):
            assert M._R(ch["columns"][1]["preagg"][40:48]).i64() == int(x["cols"][0]["values"].view(np.int64)[s])
        assert sum(struct.unpack(">I", ch["columns"][2]["preagg"])[0] for ch in p["chunks"]) == mi["rows_after_merge"] == info["n_rows"]
    finally:
        merged.close()
        ordered_only.close()
        if back:
            back.close()


def test_downsample_result_writes_and_reopens():
    src = Shard.synth(7, 5000, [(L.TYPE_FLOAT, L.SYNTH_F_HI, 50), (L.TYPE_INT, L.SYNTH_INT_WALK, 0), (L.TYPE_BOOL, L.SYNTH_BOOL, 100)], t0=T0, dt=SEC, seed=5)
    ds = src.downsample_shard(60 * SEC, T0, T0 + 4999 * SEC, {L.TYPE_FLOAT: ["min", "max", "sum", "count", "first", "last"], L.TYPE_INT: ["sum", "count"], L.TYPE_BOOL: ["count", "last"]})
    new = ds.open()
    back = None
    try:
        f = write_tssp(new, "ds")
        p = _check_crcs(f)
        assert [c["name"] for c in p["chunks"][0]["columns"]] == [n.encode() for n, *_ in ds.columns()[0]] + [b"time"]
        assert p["trailer"]["data_size"] == int(sum(int(pl.sum()) for _n, _t, _po, pl in ds.columns()[0]) + ds.columns()[1][1].sum()) + 4 * len(p["chunks"][0]["columns"]) * 7
        back = Shard.open_tssp(f)
        assert _referenced_pages(new.export()) == _referenced_pages(back.export())
        types = [t for _n, t, _po, _pl in ds.columns()[0]]
        assert _same_answers(new, back, types) > 20
        assert p["chunks"][0]["columns"][-1]["preagg"] == M.u32(84)       # 5000 s of rows = 84 one-minute windows
    finally:
        new.close()
        ds.close()
        src.close()
        if back:
            back.close()


# ---------------------------------------------------------------- 6: refusals
def _raises(status, fn, *text):
    with pytest.raises(L.OgpuError) as ei:
        fn()
    assert ei.value.status == status, str(ei.value)
    assert all(t in str(ei.value) for t in text), str(ei.value)


def _one_row_shard(n_seg, sids=(4,), absent=()):
    """Series of one-row segments over one integer column, pages written directly (BlockIntegerOne)."""
    ns = len(sids)
    t = T0 + np.arange(ns * n_seg, dtype=np.int64) * SEC
    rec = np.zeros((ns * n_seg, 2, 9), np.uint8)
    rec[:, :, 0] = 18
    rec[:, 0, 1:] = t.view(np.uint8).reshape(-1, 8)
    rec[:, 1, 1:] = (t // SEC).view(np.uint8).reshape(-1, 8)
    off = np.arange(ns * n_seg, dtype=np.uint64) * 18
    vlen = np.full(ns * n_seg, 9, np.uint32)
    vlen[list(absent)] = 0
    return Shard.open(rec.tobytes(), list(sids), np.arange(ns + 1) * n_seg, t, t, [("v", L.TYPE_INT, off + 9, vlen)], off, np.full(ns * n_seg, 9, np.uint32))


def test_refusals():
    sh = _one_row_shard(3, sids=(4, 9, 9))
    try:
        _raises(L.OG_E_INVAL, lambda: write_tssp(sh, "r", series=(2, 2)), "series range")
        _raises(L.OG_E_INVAL, lambda: write_tssp(sh, "r", series=(1, 4)), "series range")
        _raises(L.OG_E_INVAL, lambda: write_tssp(sh, "r"), "ascending")
        assert M.parse(write_tssp(sh, "r", series=(0, 2)))["trailer"]["id_count"] == 2
    finally:
        sh.close()
    sh = _one_row_shard(65536)
    try:
        _raises(L.OG_E_UNSUPPORTED, lambda: write_tssp(sh, "r"), "65535")
    finally:
        sh.close()
    sh = _one_row_shard(65535)
    try:
        p = _check_crcs(write_tssp(sh, "r"))                               # a fold over 65535 one-row pages
        assert len(p["chunks"][0]["tmin"]) == 65535 and p["chunks"][0]["columns"][1]["preagg"] == M.u32(65535)
    finally:
        sh.close()
    sh = _one_row_shard(4, absent=(2,))
    try:
        _raises(L.OG_E_UNSUPPORTED, lambda: write_tssp(sh, "r"), "some of its segments")
    finally:
        sh.close()
    sh = _one_row_shard(4, sids=(4, 6), absent=(4, 5, 6, 7))              # a series that lacks the column: left out of its ChunkMeta
    try:
        p = M.parse(write_tssp(sh, "r"))
        assert [[c["name"] for c in ch["columns"]] for ch in p["chunks"]] == [[b"v", b"time"], [b"time"]]
        back = Shard.open_tssp(write_tssp(sh, "r"))
        assert np.array_equal(back.export()["page_len"], sh.export()["page_len"])
        back.close()
    finally:
        sh.close()


def _be(fmt, *v):
    return np.frombuffer(struct.pack(">" + fmt, *v), np.uint8)


def test_corrupt_value_words_fail_the_write():
    """Pages that pass og_shard_open but do not hold the header's value count: a Simple8b page with a surplus value, RLE runs that
    do not add up.  The pre-aggregation pass walks every page to its end, so the write reports OG_E_CORRUPT."""
    n = 100
    t = T0 + np.arange(n, dtype=np.int64) * SEC
    tp = oracle.time_page_encode(t)
    ipage = oracle.field_page_encode(L.TYPE_INT, np.cumsum(np.random.default_rng(2).integers(-1000, 1001, n)).astype(np.int64))
    assert ipage[5] >> 4 == 2
    enc = struct.unpack(">I", ipage[6:10].tobytes())[0]
    surplus = np.concatenate([ipage[:6], _be("I", enc + 1), ipage[10:], _be("Q", 0xF << 60)])
    fpage = oracle.field_page_encode(L.TYPE_FLOAT, np.repeat([1.5, 2.5, 0.0, 7.0], n // 4))
    assert fpage[5] >> 4 == 5
    run0 = struct.unpack(">H", fpage[6:8].tobytes())[0]
    rle_n1 = np.concatenate([fpage[:6], _be("H", run0 + 1), fpage[8:]])
    for typ, page, good in ((L.TYPE_INT, surplus, ipage), (L.TYPE_FLOAT, rle_n1, fpage)):
        for pg, ok in ((good, True), (page, False)):
            data = np.concatenate([pg, tp])
            sh = Shard.open(data, [1], [0, 1], [int(t[0])], [int(t[-1])], [("v", typ, [0], [pg.size])], [pg.size], [tp.size])
            try:
                if ok:
                    _check_crcs(write_tssp(sh, "c"))
                else:
                    _raises(L.OG_E_CORRUPT, lambda: write_tssp(sh, "c"), "segment 0")
            finally:
                sh.close()
