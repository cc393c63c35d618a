"""Every device buffer the library allocates goes back to the pool when the handle that owns it is closed, or when the call
that needed it returns, refusals included.

The count is the default memory pool's current usage (CU_MEMPOOL_ATTR_USED_MEM_CURRENT, read through the driver API), read
after og_release_cached_memory(), which synchronises the device.  Every library buffer comes from that pool; torch's caching
allocator does not, and the count is per process, so other users of the GPU do not move it."""
import ctypes as C
import struct

import numpy as np
import pytest
import torch

import oracle
from opengemini_b200 import AggQuery, Shard, write_tssp
from opengemini_b200 import _lib as L
from test_gpu_out_of_order import _file_desc, _series

pytestmark = pytest.mark.gpu
T0, SEC = 1_700_000_000_000_000_000, 1_000_000_000
CU_MEMPOOL_ATTR_USED_MEM_CURRENT = 7
TYPE_STRING = 4
FULL_STRING_PAGE_TAG = 34  # EncodeColumnHeader: a string page without nulls


@pytest.fixture(scope="module", autouse=True)
def _device():
    Shard.init(0)


def _pool_used():
    L.check(L.lib().og_release_cached_memory(), "og_release_cached_memory")
    cu = C.CDLL("libcuda.so.1")
    dev, pool, used = C.c_int(), C.c_void_p(), C.c_uint64()
    assert cu.cuInit(0) == 0
    assert cu.cuDeviceGet(C.byref(dev), 0) == 0
    assert cu.cuDeviceGetDefaultMemPool(C.byref(pool), dev) == 0
    assert cu.cuMemPoolGetAttribute(pool, CU_MEMPOOL_ATTR_USED_MEM_CURRENT, C.byref(used)) == 0
    return used.value


class _NoLeak:
    """with _NoLeak(): ... asserts that the block leaves the pool's usage where it found it"""

    def __enter__(self):
        self.before = _pool_used()
        return self

    def __exit__(self, typ, *_):
        if typ is None:
            after = _pool_used()
            assert after == self.before, f"{after - self.before} bytes of device memory still in use"


def _synth(n_series=64, rows=3000):
    return Shard.synth(n_series, rows, [(L.TYPE_FLOAT, L.SYNTH_F_HI, 0), (L.TYPE_FLOAT, L.SYNTH_F_LO, 5), (L.TYPE_INT, L.SYNTH_INT_WALK, 0)],
                       t0=T0, dt=SEC, seed=7)


def _desc(sids, rows, t_first, seed, n=500, decimals=None):
    """Shard.desc of float series (one column "v"), `rows` rows each at 1 s from t_first, in segments of n rows"""
    rng = np.random.default_rng(seed)
    pages, tpages, tmins, tmaxs, ssb = [], [], [], [], [0]
    for _ in sids:
        v = 100.0 + rng.random(rows) * 5
        if decimals is not None:
            v = np.round(v, decimals)
        for g in range(0, rows, n):
            pages.append(oracle.field_page_encode(L.TYPE_FLOAT, v[g:g + n]))
            t = t_first + (np.arange(g, min(rows, g + n), dtype=np.int64)) * SEC
            tpages.append(oracle.time_page_encode(t)); tmins.append(t[0]); tmaxs.append(t[-1])
        ssb.append(len(pages))
    blob, offs, lens, pos = [], [], [], 0
    for p in pages + tpages:
        offs.append(pos); lens.append(p.size); blob.append(p); pos += p.size
    nseg = len(pages)
    data = np.concatenate(blob)
    return data, Shard.desc(data, np.asarray(sids), ssb, tmins, tmaxs, [("v", L.TYPE_FLOAT, offs[:nseg], lens[:nseg])], offs[nseg:], lens[nseg:])


# (calls, flags, group, og_stats.path) on _synth(): 0 tile, 1 general fused, 2 / 3 lane-interleaved (per-series / folded cells),
# 4 k_fused_multi, 5 k_fused_cols
PATHS = [
    ([("sum", 0), ("max", 0)], L.Q_NO_FUSED, "all", 0),
    ([("sum", 2), ("min", 2)], 0, "all", 1),
    ([("sum", 0), ("count", 0)], L.Q_STRICT_ORDER, "all", 2),
    ([("sum", 0), ("max", 0)], 0, "series", 2),
    ([("sum", 0), ("count", 0)], 0, "all", 3),
    ([("sum", 0), ("last", 1)], L.Q_NO_FAST, "all", 4),
    ([("sum", 0), ("sum", 1), ("count", 2)], 0, "all", 5),
]


def test_queries_on_every_path_release_their_buffers():
    with _NoLeak():
        sh = _synth()
        for calls, flags, group, path in PATHS:
            q = AggQuery(sh, calls, 60 * SEC, T0, T0 + 2999 * SEC, flags=flags, group=group)
            for _ in range(2):
                st = q.run().stats()
                assert st["path"] == path, (calls, flags, group)
            q.dense_host()
            q.close()
        sh.close()  # the lane-interleaved copy stays cached in the shard until here


def test_synth_and_decode_release_their_buffers():
    with _NoLeak():
        sh = _synth(8, 2500)
        for seg in (0, 5):
            for desc in (False, True):
                sh.decode_segment(seg, descending=desc)
        nseg = sh.info()["n_segments"]
        vals = torch.zeros(nseg * 1000, dtype=torch.float64, device="cuda")
        rows = torch.zeros(nseg, dtype=torch.int32, device="cuda")
        L.check(L.lib().og_decode_column_device(sh.h, 0, 0, nseg, vals.data_ptr(), 8000, rows.data_ptr()), "og_decode_column_device")
        assert int(rows.sum()) == 8 * 2500
        sh.close()


def test_encode_pages_releases_its_scratch():
    rng = np.random.default_rng(8)
    nseg, rps = 5, 1000
    fv = torch.from_numpy(np.cumsum(rng.integers(-3, 4, nseg * rps)).astype(np.float64)).cuda()
    iv = torch.from_numpy(rng.integers(-50, 50, nseg * rps)).cuda()
    valid = torch.from_numpy((rng.random(nseg * rps) > 0.1).astype(np.uint8)).cuda()
    rows = torch.full((nseg,), rps, dtype=torch.int32, device="cuda")
    out = torch.zeros(nseg * 8704, dtype=torch.uint8, device="cuda")
    off = torch.zeros(nseg, dtype=torch.int64, device="cuda")
    ln = torch.zeros(nseg, dtype=torch.int32, device="cuda")
    total = C.c_uint64()
    with _NoLeak():
        L.check(L.lib().og_encode_pages(L.TYPE_FLOAT, 0, fv.data_ptr(), None, None, nseg, rps, out.data_ptr(), out.numel(),
                                        off.data_ptr(), ln.data_ptr(), C.byref(total)), "og_encode_pages")
        L.check(L.lib().og_encode_pages(L.TYPE_INT, 0, iv.data_ptr(), valid.data_ptr(), rows.data_ptr(), nseg, rps, out.data_ptr(), out.numel(),
                                        off.data_ptr(), ln.data_ptr(), C.byref(total)), "og_encode_pages")


@pytest.mark.parametrize("out_of_order", [False, True])
def test_open_files_releases_the_file_set(out_of_order):
    _da, a = _desc([1, 2, 3], 2000, T0, seed=1)
    # out of order: rows inside the ordered file's range; ordered: the next 2000 s
    _db, b = _desc([2, 3, 4], 800, T0 + (500 if out_of_order else 2000) * SEC, seed=2)
    with _NoLeak():
        sh = Shard.open_files([(a, False), (b, out_of_order)])
        assert (sh.merge_info()["series_merged"] > 0) == out_of_order
        q = AggQuery(sh, [("sum", 0), ("count", 0)], 60 * SEC, T0, T0 + 3000 * SEC).run()
        q.close()
        sh.close()


def test_append_flush_and_compaction_release_what_they_replace():
    """One shard through every rewrite, each after a query that built the lane-interleaved copy of the layout it replaces, and each
    refused once on the way: the copies, the old state and the passes' scratch all go back to the pool."""
    n = 3000
    t = T0 + np.arange(n, dtype=np.int64) * SEC
    ok = np.ones(n, bool)
    rng = np.random.default_rng(12)
    # sid 1 holds string values in full segments: a re-cut at 700 rows reaches them, one at 1000 rows leaves the series alone
    base = {1: _series(t, {"v": (L.TYPE_FLOAT, 100 + rng.random(n), ok), "s": (TYPE_STRING, None, ok)}),
            2: _series(t, {"v": (L.TYPE_FLOAT, 100 + rng.random(n), ok)})}
    late_t = T0 + np.arange(500, 900, dtype=np.int64) * SEC + SEC // 2
    late = {2: _series(late_t, {"v": (L.TYPE_FLOAT, 100 + rng.random(late_t.size), np.ones(late_t.size, bool))})}
    rows_t = np.concatenate([T0 + np.arange(1000, 1100, dtype=np.int64) * SEC + SEC // 4, T0 + np.arange(n, n + 700, dtype=np.int64) * SEC])
    rows = {2: _series(rows_t, {"v": (L.TYPE_FLOAT, 100 + rng.random(rows_t.size), np.ones(rows_t.size, bool))})}

    def query(sh):
        q = AggQuery(sh, [("sum", 1), ("count", 1)], 60 * SEC, T0, T0 + (n + 700) * SEC).run()
        assert q.stats()["il_state"] == 1
        return q

    def refused(status, text, call):
        with pytest.raises(L.OgpuError) as ei:
            call()
        assert ei.value.status == status and text in str(ei.value), str(ei.value)

    with _NoLeak():
        sh = Shard.open_files([(_file_desc(base), False)])
        q = query(sh)
        refused(L.OG_E_STATE, "before appending files", lambda: sh.append_files([(_file_desc(late), True)]))
        q.close()
        sh.append_files([(_file_desc(late), True)])
        assert sh.merge_info()["series_merged"] == 1
        q = query(sh)
        refused(L.OG_E_STATE, "before appending rows", lambda: sh.append_rows(rows))
        q.close()
        assert sh.append_rows(rows)["out_of_order_rows"] == 100
        q = query(sh)
        refused(L.OG_E_STATE, "before compacting it", lambda: sh.compact())
        q.close()
        refused(L.OG_E_UNSUPPORTED, "string column", lambda: sh.compact(700))
        assert sh.compact()["series_rewritten"] == 1
        query(sh).close()
        sh.close()


def test_downsample_and_tssp_write_release_their_buffers():
    with _NoLeak():
        sh = _synth(16, 3000)
        ds = sh.downsample(0, 60 * SEC, T0, T0 + 2999 * SEC)
        reopened = ds.open()
        assert len(write_tssp(reopened, "m")) > 0
        reopened.close()
        ds.close()
        ds = sh.downsample_shard(60 * SEC, T0, T0 + 2999 * SEC, {L.TYPE_FLOAT: ["min", "max", "sum", "count"], L.TYPE_INT: ["sum", "last"]})
        assert ds.rows > 0
        ds.close()
        assert len(write_tssp(sh, "m")) > 0
        sh.close()


def test_corrupt_page_at_open_releases_the_half_built_shard():
    n = 100
    t = T0 + np.arange(n, dtype=np.int64) * SEC
    tp = oracle.time_page_encode(t)
    bad = oracle.field_page_encode(L.TYPE_FLOAT, 100 + np.random.default_rng(1).random(n)).copy()
    bad[5] = 0x70  # no float block tag
    with _NoLeak():
        with pytest.raises(L.OgpuError) as ei:
            Shard.open(np.concatenate([bad, tp]), [1], [0, 1], [int(t[0])], [int(t[-1])], [("v", L.TYPE_FLOAT, [0], [bad.size])], [bad.size], [tp.size])
        assert ei.value.status == L.OG_E_CORRUPT


def test_snappy_pages_in_caller_device_memory_are_refused_without_a_leak():
    data, d = _desc([1, 2], 1000, T0, seed=5, decimals=2)  # few decimals: the encoder stores the blocks as Snappy
    dev = torch.zeros(data.size + 1024, dtype=torch.uint8, device="cuda")
    dev[:data.size] = torch.from_numpy(data).cuda()
    d.data = C.cast(C.c_void_p(dev.data_ptr()), L.u8p)
    d.flags = L.SHARD_DEVICE_DATA
    with _NoLeak():
        with pytest.raises(L.OgpuError) as ei:
            Shard.open_desc(d)
        assert ei.value.status == L.OG_E_UNSUPPORTED and "Snappy" in str(ei.value)


def test_refused_plan_releases_the_query():
    """a string count over more than OG_MULTI_MAXC (4) columns is refused when k_fused_cols does not take the query"""
    n, segs, n_float = 100, 2, 4
    t_pages, f_pages, s_pages, tmins, tmaxs = [], [[] for _ in range(n_float)], [], [], []
    rng = np.random.default_rng(4)
    for _series in range(2):
        for g in range(segs):
            t = T0 + (np.arange(n, dtype=np.int64) + g * n) * SEC
            t_pages.append(oracle.time_page_encode(t)); tmins.append(t[0]); tmaxs.append(t[-1])
            s_pages.append(np.frombuffer(bytes([FULL_STRING_PAGE_TAG]) + struct.pack(">I", n) + b"\x10opaque", np.uint8))
            for k in range(n_float):
                f_pages[k].append(oracle.field_page_encode(L.TYPE_FLOAT, rng.random(n)))
    blob, pos, cols = [], 0, []

    def place(pages):
        nonlocal pos
        offs, lens = [], []
        for p in pages:
            offs.append(pos); lens.append(p.size); blob.append(p); pos += p.size
        return offs, lens

    cols.append(("s", TYPE_STRING, *place(s_pages)))
    for k in range(n_float):
        cols.append((f"f{k}", L.TYPE_FLOAT, *place(f_pages[k])))
    toff, tlen = place(t_pages)
    with _NoLeak():
        sh = Shard.open(np.concatenate(blob), [1, 2], [0, segs, 2 * segs], tmins, tmaxs, cols, toff, tlen)
        q = AggQuery(sh, [("count", 0)] + [("sum", 1 + k) for k in range(n_float)], 60 * SEC, T0, T0 + segs * n * SEC, flags=L.Q_NO_FAST)
        with pytest.raises(L.OgpuError) as ei:
            q.run()
        assert ei.value.status == L.OG_E_UNSUPPORTED
        q.close()
        sh.close()
