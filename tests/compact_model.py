"""CPU model of og_shard_compact, built only from the oracle and numpy: from a shard's export, the directory and page bytes the
compacted shard must hold.

  1. per series, from the directory alone (rows and page lengths per segment): where the re-cut starts (`recut_start`)
       - nowhere when every segment but the last holds R rows, the last 1..R, and every column has a page in every segment or none
       - at the first segment when a column has pages in only some segments
       - else at the first segment that is not the last and holds fewer than R rows, or holds more than R
  2. the rows from there on decoded with oracle.time_page_decode / field_page_decode (null where a segment has no page)
  3. cut into segments of R rows, the remainder last; every column of the series gets a page in each, from the oracle's encoders
     (a float segment the Gorilla encoder refuses, +Inf and -Inf in one segment, gets the raw page [header][0x00][values LE], and
     an int segment the reference would hand to zstd, a zig-zag delta above 2^60 - 1, the raw page [header][0x40][u32 BE 8n][zig-zag
     BE values], int.go uncompressedData);
     a string column, which must be null in every re-cut row, gets the all-null page [44][u32 BE rows]

The device encoders write a raw page where the reference takes Snappy (NaN, few decimals: DESIGN.md "Deviations"), so byte
comparisons against this model use values that stay clear of that route.
"""
import struct

import numpy as np

import oracle
from opengemini_b200 import _lib as L

TYPE_STRING = 4


class StringValues(ValueError):
    """a string column holds a value inside a re-cut range"""


def recut_start(rows, present, R):
    """rows: the row count of each segment of one series; present: [segment][column] has a page.  -> the first re-cut segment,
    or None when the series is compact."""
    if len(rows) == 0:
        return None
    present = np.asarray(present, bool).reshape(len(rows), -1)
    if (present.any(axis=0) != present.all(axis=0)).any():
        return 0
    for j, r in enumerate(rows):
        if r > R or (j + 1 < len(rows) and r < R):
            return j
    return None


def cut(n_rows, R):
    """segment row counts of n_rows re-cut rows"""
    return [min(R, n_rows - a) for a in range(0, n_rows, R)]


def _header(typ, valid):
    rows, nil = valid.size, int(valid.size - valid.sum())
    full = {L.TYPE_FLOAT: 31, L.TYPE_INT: 32, L.TYPE_BOOL: 33}[typ]
    if nil == 0:
        return bytes([full]) + struct.pack(">I", rows)
    if nil == rows:
        return bytes([full + 10]) + struct.pack(">I", rows)
    bm = np.packbits(valid.astype(np.uint8), bitorder="little").tobytes()
    return bytes([typ]) + struct.pack(">I", len(bm)) + bm + struct.pack(">II", 0, nil)


def raw_float_page(values, valid):
    """the encoders' raw page for a float segment: header, 0x00, the non-null values little-endian"""
    return np.frombuffer(_header(L.TYPE_FLOAT, valid) + b"\x00" + np.ascontiguousarray(values[valid], "<f8").tobytes(), np.uint8)


def zigzag_be(values):
    """int64 values -> their zig-zag encodings as big-endian bytes (MarshalInt64Append)"""
    v = np.asarray(values, np.int64)
    return ((v.astype(np.uint64) << np.uint64(1)) ^ (v >> np.int64(63)).astype(np.uint64)).astype(">u8").tobytes()


def raw_int_page(values, valid):
    """the encoders' raw page for an int segment: header, 0x40, u32 BE 8n, the non-null values zig-zag big-endian"""
    v = np.asarray(values, np.int64)[valid]
    return np.frombuffer(_header(L.TYPE_INT, valid) + struct.pack(">BI", 0x40, 8 * v.size) + zigzag_be(v), np.uint8)


def encode_field(typ, values, valid):
    if typ == TYPE_STRING:
        return np.frombuffer(bytes([44]) + struct.pack(">I", valid.size), np.uint8)
    try:
        return oracle.field_page_encode(typ, np.ascontiguousarray(values), None if valid.all() else valid.astype(np.uint8))
    except ValueError:
        if typ == L.TYPE_FLOAT:
            return raw_float_page(values, valid)
        if typ == L.TYPE_INT:  # the oracle does not restate zstd: the device writes the raw block there
            return raw_int_page(values, valid)
        raise


def _page(ex, c, g):
    o, n = int(ex["page_off"][c][g]), int(ex["page_len"][c][g])
    return ex["data"][o:o + n]


def decode_segment(ex, g):
    """(times, [(values per row, valid per row)] per column) of segment g; strings: valid from the page header only"""
    nc = ex["col_types"].size
    t = oracle.time_page_decode(_page(ex, nc, g), cap=1 << 17)
    cols = []
    for c in range(nc):
        typ = int(ex["col_types"][c])
        dt = np.uint8 if typ == L.TYPE_BOOL else np.float64 if typ == L.TYPE_FLOAT else np.int64
        v, ok = np.zeros(t.size, dt), np.zeros(t.size, bool)
        p = _page(ex, c, g)
        if p.size and typ == TYPE_STRING:
            if p[0] != 44:
                raise StringValues(c)
        elif p.size:
            vals, ok = oracle.field_page_decode(typ, p, cap=t.size + 8)
            v[ok] = vals
        cols.append((v, ok))
    return t, cols


def plan(ex, R):
    """[(series, first re-cut segment)] for every series that is not compact"""
    nc = ex["col_types"].size
    ssb = ex["series_seg_begin"]
    rows = [oracle.time_page_decode(_page(ex, nc, g), cap=1 << 17).size for g in range(ex["seg_tmin"].size)]
    out = []
    for u in range(ssb.size - 1):
        a, b = int(ssb[u]), int(ssb[u + 1])
        k = recut_start(rows[a:b], ex["page_len"][:nc, a:b].T > 0, R)
        if k is not None:
            out.append((u, a + k))
    return out, rows


def expected(ex, R=1000):
    """The compacted shard: dict(series_seg_begin, seg_tmin, seg_tmax, pages [segment][column + time] (np.uint8 or None for no
    page), info counters).  Raises StringValues when a string column holds a value in a re-cut range, ValueError when times do not
    strictly ascend there."""
    nc = ex["col_types"].size
    spans, _rows = plan(ex, R)
    first = dict(spans)
    ssb, tmin, tmax, pages = [0], [], [], []
    info = dict(series_rewritten=0, segments_kept=0, segments_rewritten_in=0, segments_rewritten_out=0, rows_rewritten=0)
    for u in range(ex["series_seg_begin"].size - 1):
        a, b = int(ex["series_seg_begin"][u]), int(ex["series_seg_begin"][u + 1])
        k = first.get(u, b)
        for g in range(a, k):
            pages.append([_page(ex, c, g) if ex["page_len"][c][g] else None for c in range(nc + 1)])
            tmin.append(int(ex["seg_tmin"][g])); tmax.append(int(ex["seg_tmax"][g]))
        if k < b:
            mask = (ex["page_len"][:nc, a:b] > 0).any(axis=1)
            segs = [decode_segment(ex, g) for g in range(k, b)]
            t = np.concatenate([s[0] for s in segs])
            if t.size > 1 and not (np.diff(t) > 0).all():
                raise ValueError(f"times do not strictly ascend in series {u}")
            cols = [(np.concatenate([s[1][c][0] for s in segs]), np.concatenate([s[1][c][1] for s in segs])) for c in range(nc)]
            for c in range(nc):
                if int(ex["col_types"][c]) == TYPE_STRING and cols[c][1].any():
                    raise StringValues(c)
            lo = 0
            for n in cut(t.size, R):
                seg = []
                for c in range(nc):
                    v, ok = cols[c]
                    seg.append(encode_field(int(ex["col_types"][c]), v[lo:lo + n], ok[lo:lo + n]) if mask[c] else None)
                seg.append(oracle.time_page_encode(np.ascontiguousarray(t[lo:lo + n])))
                pages.append(seg)
                tmin.append(int(t[lo])); tmax.append(int(t[lo + n - 1]))
                lo += n
            info["series_rewritten"] += 1
            info["segments_rewritten_in"] += b - k
            info["segments_rewritten_out"] += len(cut(t.size, R))
            info["rows_rewritten"] += t.size
        info["segments_kept"] += k - a
        ssb.append(len(tmin))
    if info["series_rewritten"] == 0:
        info["segments_kept"] = 0
    return dict(series_seg_begin=np.array(ssb, np.uint32), seg_tmin=np.array(tmin, np.int64), seg_tmax=np.array(tmax, np.int64),
                pages=pages, info=info)


def assert_matches(ex, want):
    """a compacted shard's export against expected(...): directory and every page's bytes"""
    assert np.array_equal(ex["series_seg_begin"], want["series_seg_begin"])
    assert np.array_equal(ex["seg_tmin"], want["seg_tmin"])
    assert np.array_equal(ex["seg_tmax"], want["seg_tmax"])
    nc1 = ex["page_off"].shape[0]
    for g, seg in enumerate(want["pages"]):
        for c in range(nc1):
            got = _page(ex, c, g)
            if seg[c] is None:
                assert got.size == 0, (g, c)
            else:
                assert np.array_equal(got, np.asarray(seg[c], np.uint8)), (g, c, got.size, len(seg[c]))
