"""tests/tssp_write_model.py (the Python restatement of the reference's TSSP writer that og_shard_write_tssp is compared with)
against hand-worked cases, and the new entry points in the ABI.  No GPU needed."""
import ctypes
import math
import os
import struct
import zlib

from opengemini_b200 import _lib as L

import tssp_write_model as M

NAN = float("nan")


def _blob6(b, is_float):
    enc = M.f64 if is_float else M.i64
    return enc(b.minv) + enc(b.maxv) + M.i64(b.mint) + M.i64(b.maxt) + enc(b.sum) + M.i64(b.count)


def test_new_entry_points_are_exported():
    lib = ctypes.CDLL(L.LIB_PATH)
    for sym in ("og_shard_write_tssp", "og_tssp_image_size", "og_tssp_image_export", "og_tssp_image_timing", "og_tssp_image_free"):
        assert sym in L.EXPORTS and hasattr(lib, sym), sym


def test_write_refuses_null_arguments_without_a_device():
    h = ctypes.c_void_p()
    assert L.lib().og_shard_write_tssp(None, None, ctypes.byref(h)) == L.OG_E_INVAL
    assert L.lib().og_last_error()


def test_one_row_column_uses_the_16_byte_form():
    b = M.preagg(M.TYPE_FLOAT, [([2.5], [1], [77])])
    assert b.marshal() == M.f64(2.5) + M.i64(77) and len(b.marshal()) == 16
    b = M.preagg(M.TYPE_INT, [([0, -9, 0], [0, 1, 0], [5, 6, 7])])
    assert (b.minv, b.mint, b.maxv, b.maxt, b.sum, b.count) == (-9, 6, -9, 6, -9, 1)
    assert b.marshal() == M.i64(-9) + M.i64(6)


def test_all_null_column_keeps_the_initial_values():
    b = M.preagg(M.TYPE_INT, [([0, 0], [0, 0], [1, 2])])
    assert b.marshal() == _blob6(b, False) and (b.minv, b.maxv, b.mint, b.maxt, b.sum, b.count) == (M.MAX_I64, M.MIN_I64, 0, 0, 0, 0)
    b = M.preagg(M.TYPE_FLOAT, [([0.0], [0], [1])])
    assert (b.minv, b.maxv, b.mint, b.maxt, b.sum, b.count) == (M.MAX_F64, -M.MAX_F64, 0, 0, 0.0, 0)
    assert M.preagg(M.TYPE_STRING, [([None, None], [0, 0], [1, 2])]).marshal() == M.i64(0)


def test_nan_never_becomes_min_or_max():
    b = M.preagg(M.TYPE_FLOAT, [([NAN, 3.0, 1.0, NAN], [1, 1, 1, 1], [10, 20, 30, 40])])
    assert (b.minv, b.mint, b.maxv, b.maxt, b.count) == (1.0, 30, 3.0, 20, 4) and math.isnan(b.sum)
    b = M.preagg(M.TYPE_FLOAT, [([NAN], [1], [10]), ([NAN], [1], [20])])
    assert (b.minv, b.mint, b.maxv, b.maxt, b.count) == (M.MAX_F64, 0, -M.MAX_F64, 0, 2)
    b = M.preagg(M.TYPE_FLOAT, [([NAN], [1], [10])])  # one value: the 16-byte form carries the untouched initial min and time 0
    assert b.marshal() == M.f64(M.MAX_F64) + M.i64(0)


def test_max_float_equals_the_initial_value_and_is_not_recorded():
    b = M.preagg(M.TYPE_FLOAT, [([M.MAX_F64, M.MAX_F64], [1, 1], [10, 20])])
    assert (b.minv, b.mint) == (M.MAX_F64, 0) and (b.maxv, b.maxt) == (M.MAX_F64, 10)
    b = M.preagg(M.TYPE_FLOAT, [([-M.MAX_F64, -M.MAX_F64], [1, 1], [10, 20])])
    assert (b.maxv, b.maxt) == (-M.MAX_F64, 0) and (b.minv, b.mint) == (-M.MAX_F64, 10)


def test_signed_zeros_first_occurrence_wins():
    b = M.preagg(M.TYPE_FLOAT, [([0.0, -0.0], [1, 1], [10, 20])])
    assert (b.mint, b.maxt) == (10, 10) and math.copysign(1, b.minv) == 1 and math.copysign(1, b.maxv) == 1
    b = M.preagg(M.TYPE_FLOAT, [([-0.0, 0.0], [1, 1], [10, 20])])
    assert (b.mint, b.maxt) == (10, 10) and math.copysign(1, b.minv) == -1 and struct.pack(">d", b.sum) == struct.pack(">d", 0.0)


def test_bool_time_is_indexed_by_value_not_by_row():
    # rows: null, null, true, false at times 10..40.  Values [1, 0]: max 1 is value 0 -> times[0] = 10, min 0 is value 1 -> times[1] = 20
    b = M.preagg(M.TYPE_BOOL, [([0, 0, 1, 0], [0, 0, 1, 1], [10, 20, 30, 40])])
    assert (b.minv, b.mint, b.maxv, b.maxt, b.count) == (0, 20, 1, 10, 2)
    assert b.marshal() == M.i64(2) + M.i64(20) + M.i64(10) + b"\x00\x01" and len(b.marshal()) == 26
    # per segment: the index restarts with each segment's times
    b = M.preagg(M.TYPE_BOOL, [([1], [1], [10]), ([0, 0], [0, 1], [20, 30])])
    assert (b.minv, b.mint, b.maxv, b.maxt) == (0, 20, 1, 10)
    assert M.preagg(M.TYPE_BOOL, [([0], [0], [1])]).marshal() == M.i64(0) + M.i64(0) + M.i64(0) + b"\x02\xff"


def test_float_sum_is_sequential_across_segments():
    vals = [1e16, 1.0, 1.0, 1.0, 1.0]
    seq = 0.0
    for v in vals:
        seq += v
    pairwise = (vals[0] + vals[1]) + ((vals[2] + vals[3]) + vals[4])
    per_segment = (vals[0] + vals[1] + vals[2]) + (vals[3] + vals[4])
    assert seq != pairwise and seq != per_segment
    b = M.preagg(M.TYPE_FLOAT, [(vals[:3], [1] * 3, [1, 2, 3]), (vals[3:], [1] * 2, [4, 5])])
    assert struct.pack(">d", b.sum) == struct.pack(">d", seq)


def test_int_sum_wraps():
    b = M.preagg(M.TYPE_INT, [([M.MAX_I64, 1], [1, 1], [1, 2])])
    assert b.sum == M.MIN_I64


def test_xxhash64_known_values():
    assert M.xxh64(b"") == 0xEF46DB3751D8E999
    assert M.xxh64(b"a") == 0xD24EC4F1A98C6E5B
    assert M.xxh64(b"abc") == 0x44BC2CF5AD770999
    assert M.xxh64(b"Nobody inspects the spammish repetition") == 0xFBCEA83C8A378BF1


def test_bloom_filter_holds_every_sid():
    sids = list(range(7, 7 + 300, 3))
    bits, m, k = M.bloom(sids)
    assert len(bits) & (len(bits) - 1) == 0 and len(bits) * 8 >= m and k >= 1
    for sid in sids:
        key = struct.pack(">Q", sid)
        h0, h1 = M.xxh64(key), M.xxh64(key[:-1] + b"\x00")
        assert all(bits[((h0 + h1 * i) & (len(bits) * 8 - 1)) >> 3] >> (((h0 + h1 * i) & (len(bits) * 8 - 1)) & 7) & 1 for i in range(k))
    assert M.bloom([1])[0] == M.bloom([1])[0] and len(M.bloom([1])[0]) == 8


def _chunks(n_series):
    chunks = []
    for i in range(n_series):
        times = [[100 * i + k for k in range(3)], [100 * i + 50]]
        cols = [(b"f", M.TYPE_FLOAT, [b"PAGE-f0-%d" % i, b"p1"], [([1.0, 2.0, 0.5], [1, 1, 1]), ([4.0], [1])]),
                (b"i", M.TYPE_INT, [b"x", b"PAGE-i1"], [([5, 0, 7], [1, 0, 1]), ([0], [0])])]
        if i % 3 == 0:
            cols = cols[:1]
        chunks.append(dict(sid=10 + 2 * i, tmin=[t[0] for t in times], tmax=[t[-1] for t in times], times=times,
                           time_pages=[b"T0", b"T1-%d" % i], columns=cols))
    return chunks


def test_model_file_parses_back_to_its_inputs():
    chunks = _chunks(1200)  # three chunk-meta blocks of at most 512
    f = M.build(chunks, b"cpu_meas")
    p = M.parse(f)
    t = p["trailer"]
    assert t["name"] == b"cpu_meas" and t["id_count"] == 1200 and (t["min_id"], t["max_id"]) == (10, 10 + 2 * 1199)
    assert t["flags"] == 1 | (10 << 32) and t["data_off"] == 16
    assert (t["min_time"], t["max_time"]) == (0, 100 * 1199 + 50)
    assert [m["count"] for m in p["meta_index"]] == [512, 512, 176] and [m["id"] for m in p["meta_index"]] == [10, 10 + 1024, 10 + 2048]
    assert len(p["chunks"]) == 1200
    end = 16
    for ch, got in zip(chunks, p["chunks"]):
        assert got["sid"] == ch["sid"] and got["offset"] == end and got["tmin"] == ch["tmin"] and got["tmax"] == ch["tmax"]
        want_cols = [(n, ty, pg) for n, ty, pg, _r in ch["columns"]] + [(b"time", M.TYPE_INT, ch["time_pages"])]
        assert [(c["name"], c["type"]) for c in got["columns"]] == [(n, ty) for n, ty, _pg in want_cols]
        for c, (_n, _ty, pages) in zip(got["columns"], want_cols):
            assert [f[o:o + z] for o, z in c["segs"]] == pages
            assert c["crc"] == zlib.crc32(b"".join(pages))
        assert got["columns"][-1]["preagg"] == M.u32(4)
        assert got["columns"][0]["preagg"] == M.f64(0.5) + M.f64(4.0) + M.i64(ch["times"][0][2]) + M.i64(ch["times"][1][0]) + M.f64(7.5) + M.i64(4)
        end += got["size"]
    assert end == 16 + t["data_size"]
    assert p["bloom"] == M.bloom([c["sid"] for c in chunks])[0]
    assert p["id_time"][:8] == M.u32(1200) + M.u32(1)


def test_the_product_does_not_import_the_model():
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    for dirpath, _, files in os.walk(os.path.join(root, "opengemini_b200")):
        for fn in files:
            if fn.endswith((".py", ".cu", ".cuh", ".h", ".cpp")):
                assert "tssp_write_model" not in open(os.path.join(dirpath, fn), errors="replace").read()
