"""The span rule of og_shard_compact on hand-worked cases, the model's re-cut on host-built shards, and the og_compact_desc /
og_compact_info layouts against include/ogpu.h (no GPU needed)."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import compact_model as cm
import oracle
import segment_shards as ss
from opengemini_b200 import _lib as L

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _all(rows, nc=2):
    return np.ones((len(rows), nc), bool)


# ---------------------------------------------------------------- which segment the re-cut starts at
@pytest.mark.parametrize("rows, present, R, want", [
    ([1000, 1000, 437], None, 1000, None),                 # already compact
    ([1000], None, 1000, None),
    ([5], None, 1000, None),                               # one short segment is its own last one
    ([700, 700, 700], None, 1000, 0),                      # every segment short
    ([700, 700, 700], None, 700, None),                    # ... and compact at R = 700
    ([1000, 1000, 437, 5, 5, 5], None, 1000, 2),           # flushes after a short tail: from the tail on
    ([4096], None, 1000, 0),                               # one long segment
    ([1000, 4096, 1000], None, 1000, 1),
    ([1] * 6, None, 1000, 0),                              # one-row segments
    ([1] * 6, None, 1, None),                              # ... compact at R = 1
    ([1, 2, 1], None, 1, 1),                               # R = 1: a two-row segment
    ([1000, 1000, 20], [[1, 0], [1, 1], [1, 1]], 1000, 0),  # a column present in later segments only: the whole series
    ([1000, 1000], [[1, 0], [1, 0]], 1000, None),           # a column in no segment is fine
    ([], None, 1000, None),
])
def test_recut_start(rows, present, R, want):
    p = _all(rows) if present is None else np.array(present, bool)
    assert cm.recut_start(rows, p, R) == want


def test_cut():
    assert cm.cut(2437 + 15, 1000) == [1000, 1000, 452]
    assert cm.cut(2100, 700) == [700, 700, 700]
    assert cm.cut(3, 1) == [1, 1, 1]
    assert cm.cut(999, 1000) == [999]


# ---------------------------------------------------------------- the model's re-cut of a host-built shard
def _export_of(desc, types):
    """what Shard.export() returns, from a host L.ShardDesc"""
    ng, nc = desc.n_segments, desc.n_columns
    off = np.zeros((nc + 1, ng), np.uint64); ln = np.zeros((nc + 1, ng), np.uint32)
    for c in range(nc):
        off[c] = np.ctypeslib.as_array(desc.columns[c].page_off, shape=(ng,)); ln[c] = np.ctypeslib.as_array(desc.columns[c].page_len, shape=(ng,))
    off[nc] = np.ctypeslib.as_array(desc.time_page_off, shape=(ng,)); ln[nc] = np.ctypeslib.as_array(desc.time_page_len, shape=(ng,))
    return dict(data=np.ctypeslib.as_array(desc.data, shape=(desc.data_len,)).copy(),
                sids=np.ctypeslib.as_array(desc.sids, shape=(desc.n_series,)).copy(),
                series_seg_begin=np.ctypeslib.as_array(desc.series_seg_begin, shape=(desc.n_series + 1,)).copy(),
                seg_tmin=np.ctypeslib.as_array(desc.seg_tmin, shape=(ng,)).copy(), seg_tmax=np.ctypeslib.as_array(desc.seg_tmax, shape=(ng,)).copy(),
                page_off=off, page_len=ln, col_types=np.array(types, np.int32))


@pytest.mark.parametrize("R", [1000, 7])
def test_model_recut_keeps_every_row(R):
    kinds = ["f_hi", "i_s8b", "bool"]
    types = ss.types_of(kinds)
    rng = np.random.default_rng(R)
    series = [ss.series_rows(rng, n, kinds, null_share=[0.0, 0.05, 0.4]) for n in (2452, 2100, 40)]
    lengths = [[1000, 1000, 437, 5, 5, 5], [700, 700, 700], [1] * 40]
    desc = ss.shard_desc(series, types, lengths)
    ex = _export_of(desc, types)
    want = cm.expected(ex, R)
    for u, rows in enumerate(series):
        a, b = int(want["series_seg_begin"][u]), int(want["series_seg_begin"][u + 1])
        t = np.concatenate([oracle.time_page_decode(want["pages"][g][-1], cap=2000) for g in range(a, b)])
        assert np.array_equal(t, rows["times"])
        seg_rows = [oracle.time_page_decode(want["pages"][g][-1], cap=2000).size for g in range(a, b)]
        assert all(n == R for n in seg_rows[:-1]) and 1 <= seg_rows[-1] <= R, seg_rows
        for c, typ in enumerate(types):
            got = [oracle.field_page_decode(typ, want["pages"][g][c], cap=2000) for g in range(a, b)]
            ok = np.concatenate([x[1] for x in got])
            assert np.array_equal(ok, rows["cols"][c][1])
            v = np.concatenate([x[0] for x in got])
            assert np.array_equal(np.asarray(v).astype(np.float64), rows["cols"][c][0][ok].astype(np.float64))
    if R == 1000:  # the first series keeps its two full segments byte for byte
        assert want["info"]["segments_kept"] == 2 and want["info"]["series_rewritten"] == 3
        for c in range(len(types) + 1):
            o, n = int(ex["page_off"][c][0]), int(ex["page_len"][c][0])
            assert np.array_equal(want["pages"][0][c], ex["data"][o:o + n])


def test_model_fills_a_column_missing_from_early_segments_with_nulls():
    types = [L.TYPE_FLOAT, L.TYPE_INT]
    rng = np.random.default_rng(5)
    rows = ss.series_rows(rng, 1030, ["f_hi", "i_s8b"])
    desc = ss.shard_desc([rows], types, [[1000, 30]])
    ex = _export_of(desc, types)
    ex["page_len"][1][0] = 0  # the integer column arrives with the second segment
    want = cm.expected(ex, 1000)
    assert want["info"]["series_rewritten"] == 1 and want["info"]["segments_kept"] == 0
    v, ok = oracle.field_page_decode(L.TYPE_INT, want["pages"][0][1], cap=2000)
    assert not ok[:1000].any() and ok[1000:].all()
    v2, ok2 = oracle.field_page_decode(L.TYPE_INT, want["pages"][1][1], cap=2000)
    assert ok2.all() and np.array_equal(np.concatenate([v, v2]), rows["cols"][1][0][1000:])


def test_raw_float_page_restates_the_encoders():
    v = np.array([1.0, np.inf, 2.0, -np.inf, 3.0, 4.0])
    ok = np.array([1, 1, 0, 1, 1, 1], bool)
    p = cm.raw_float_page(v, ok)
    dv, dok = oracle.field_page_decode(L.TYPE_FLOAT, p, cap=16)
    assert np.array_equal(dok, ok) and np.array_equal(dv, v[ok])


def test_raw_int_page_where_the_reference_takes_zstd():
    """a zig-zag delta above 2^60 - 1: the oracle does not restate zstd, encode_field writes the uncompressed block"""
    v = np.array([0, 1 << 59, 3, -(1 << 62), (1 << 63) - 1, -(1 << 63)], np.int64)
    ok = np.array([1, 1, 0, 1, 1, 1], bool)
    with pytest.raises(ValueError):
        oracle.field_page_encode(L.TYPE_INT, v, ok.astype(np.uint8))
    p = cm.encode_field(L.TYPE_INT, v, ok)
    assert np.array_equal(p, cm.raw_int_page(v, ok))
    nb = 1  # [2][u32 1][bitmap][u32 0][u32 1][0x40][u32 40][zig-zag BE x 5]
    assert p[0] == L.TYPE_INT and p[13 + nb] == 0x40 and int.from_bytes(p[14 + nb:18 + nb].tobytes(), "big") == 8 * 5
    dv, dok = oracle.field_page_decode(L.TYPE_INT, p, cap=16)
    assert np.array_equal(dok, ok) and np.array_equal(dv, v[ok])
    full = cm.encode_field(L.TYPE_INT, v, np.ones(6, bool))
    assert full[0] == 32 and np.array_equal(oracle.field_page_decode(L.TYPE_INT, full, cap=16)[0], v)


# ---------------------------------------------------------------- ABI
def test_compact_structs_match_the_header(tmp_path):
    pairs = {"og_compact_desc": L.CompactDesc, "og_compact_info": L.CompactInfo}
    lines = ["#include <stdio.h>", "#include <stddef.h>", f'#include "{os.path.join(ROOT, "include", "ogpu.h")}"', "int main(void) {"]
    for cname, cls in pairs.items():
        lines.append(f'  printf("{cname} %zu\\n", sizeof({cname}));')
        for fname, _t in cls._fields_:
            lines.append(f'  printf("{cname}.{fname} %zu\\n", offsetof({cname}, {fname}));')
    lines += ["  return 0;", "}"]
    src = tmp_path / "compact.c"
    src.write_text("\n".join(lines))
    exe = tmp_path / "compact"
    subprocess.run(["gcc", "-std=c11", "-o", str(exe), str(src)], check=True)
    seen = dict(line.split() for line in subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.strip().splitlines())
    for cname, cls in pairs.items():
        assert int(seen[cname]) == C.sizeof(cls), cname
        for fname, _t in cls._fields_:
            assert int(seen[f"{cname}.{fname}"]) == getattr(cls, fname).offset, f"{cname}.{fname}"
