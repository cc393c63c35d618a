"""Test infrastructure: a TSSP file WRITER with real pre-aggregation, bloom filter and id-time sections, in plain Python, restated
from the Go sources and sharing no code with opengemini_b200/csrc (the writer under test) or with tests/tssp_file.py (whose
filler sections other tests depend on):

  engine/immutable/pre_aggregation.go                  Integer/Float/Boolean/String/TimePreAgg: reset, addValues, marshal
  engine/immutable/column_builder.go:151-349           addValues is called once per segment with that segment's times
  engine/immutable/chunkdata_builder_ts.go:37-82        chunk bytes: per column [u32 BE crc32 (IEEE) of its pages][pages]
  engine/immutable/tssp_file_meta.go:566-581,228-246    ChunkMeta / ColumnMeta; :769-778 MetaIndex
  engine/immutable/msbuilder.go:308-364,1481-1500       chunk-meta blocks: closed at 512 metas or >= 256 KiB, then u32 start offsets
  engine/immutable/msbuilder.go:1336-1353               genBloomFilter; lib/util/lifted/influxdb/pkg/bloom/bloom.go; xxHash64
  engine/immutable/sequencer.go:332-390                 IdTimePairs.Marshal (integer blocks: tests/golden/pyenc.py int_block)
  engine/immutable/trailer.go:58-66, table_stat.go:35-51,125-148   trailer; msbuilder.go:1413-1425 footer

A column is described by its decoded rows, so the pre-aggregation here never reads a page.
"""
import math
import os
import struct
import sys
import zlib

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden"))
import pyenc  # noqa: E402

M64 = (1 << 64) - 1
TYPE_INT, TYPE_FLOAT, TYPE_STRING, TYPE_BOOL = 1, 3, 4, 5
MAX_F64 = sys.float_info.max
MAX_I64, MIN_I64 = (1 << 63) - 1, -(1 << 63)


def i64(v):
    return struct.pack(">Q", ((v << 1) ^ (v >> 63)) & M64)


def u64(v):
    return struct.pack(">Q", v & M64)


def u32(v):
    return struct.pack(">I", v)


def u16(v):
    return struct.pack(">H", v)


def f64(v):
    return struct.pack(">d", v)


def _wrap(v):
    v &= M64
    return v - (1 << 64) if v >> 63 else v


class IntPreAgg:
    def __init__(self):
        self.minv, self.maxv, self.mint, self.maxt, self.sum, self.count = MAX_I64, MIN_I64, 0, 0, 0, 0

    def add_values(self, cells, valid, times):
        for i, (v, ok) in enumerate(zip(cells, valid)):
            if not ok:
                continue
            v = int(v)
            if self.minv > v:
                self.minv, self.mint = v, int(times[i])
            if self.maxv < v:
                self.maxv, self.maxt = v, int(times[i])
            self.sum = _wrap(self.sum + v)
            self.count += 1

    def marshal(self):
        if self.count == 1:
            return i64(self.minv) + i64(self.mint)
        return b"".join(i64(x) for x in (self.minv, self.maxv, self.mint, self.maxt, self.sum, self.count))


class FloatPreAgg:
    def __init__(self):
        self.minv, self.maxv, self.mint, self.maxt, self.sum, self.count = MAX_F64, -MAX_F64, 0, 0, 0.0, 0

    def add_values(self, cells, valid, times):
        for i, (v, ok) in enumerate(zip(cells, valid)):
            if not ok:
                continue
            v = float(v)
            if self.minv > v:                       # false for NaN
                self.minv, self.mint = v, int(times[i])
            if self.maxv < v:
                self.maxv, self.maxt = v, int(times[i])
            self.sum += v                           # row order, one IEEE add per value
            self.count += 1

    def marshal(self):
        if self.count == 1:
            return f64(self.minv) + i64(self.mint)
        return f64(self.minv) + f64(self.maxv) + i64(self.mint) + i64(self.maxt) + f64(self.sum) + i64(self.count)


class BoolPreAgg:
    def __init__(self):
        self.count, self.mint, self.maxt, self.minv, self.maxv = 0, 0, 0, 2, -1

    def add_values(self, cells, valid, times):
        values = [int(bool(v)) for v, ok in zip(cells, valid) if ok]
        for i, v in enumerate(values):              # times[i]: indexed by VALUE, as the reference does
            if self.minv > v:
                self.minv, self.mint = v, int(times[i])
            if self.maxv < v:
                self.maxv, self.maxt = v, int(times[i])
        self.count += len(values)

    def marshal(self):
        return i64(self.count) + i64(self.mint) + i64(self.maxt) + bytes([self.minv & 0xFF, self.maxv & 0xFF])


class StringPreAgg:
    def __init__(self):
        self.count = 0

    def add_values(self, cells, valid, times):
        self.count += sum(1 for ok in valid if ok)

    def marshal(self):
        return i64(self.count)


class TimePreAgg:
    def __init__(self):
        self.count = 0

    def add_values(self, cells, valid, times):
        self.count += len(times)

    def marshal(self):
        return u32(self.count)


BUILDERS = {TYPE_INT: IntPreAgg, TYPE_FLOAT: FloatPreAgg, TYPE_BOOL: BoolPreAgg, TYPE_STRING: StringPreAgg}


def preagg(typ, segments):
    """segments: [(cells per row, valid per row, times per row)] of one column of one chunk -> builder."""
    b = BUILDERS[typ]()
    for cells, valid, times in segments:
        b.add_values(cells, valid, times)
    return b


# ---- xxHash64 (seed 0), any length ----
_P1, _P2, _P3, _P4, _P5 = 11400714785074694791, 14029467366897019727, 1609587929392839161, 9650029242287828579, 2870177450012600261


def _rotl(x, r):
    return ((x << r) | (x >> (64 - r))) & M64


def _round(acc, inp):
    return (_rotl((acc + inp * _P2) & M64, 31) * _P1) & M64


def xxh64(data):
    n, p = len(data), 0
    if n >= 32:
        v = [(_P1 + _P2) & M64, _P2, 0, (-_P1) & M64]
        while p + 32 <= n:
            for k in range(4):
                v[k] = _round(v[k], struct.unpack_from("<Q", data, p + 8 * k)[0])
            p += 32
        h = (_rotl(v[0], 1) + _rotl(v[1], 7) + _rotl(v[2], 12) + _rotl(v[3], 18)) & M64
        for k in range(4):
            h = ((h ^ _round(0, v[k])) * _P1 + _P4) & M64
    else:
        h = _P5
    h = (h + n) & M64
    while p + 8 <= n:
        h = (_rotl(h ^ _round(0, struct.unpack_from("<Q", data, p)[0]), 27) * _P1 + _P4) & M64
        p += 8
    if p + 4 <= n:
        h = (_rotl(h ^ (struct.unpack_from("<I", data, p)[0] * _P1 & M64), 23) * _P2 + _P3) & M64
        p += 4
    while p < n:
        h = (_rotl(h ^ (data[p] * _P5 & M64), 11) * _P1) & M64
        p += 1
    h ^= h >> 33
    h = (h * _P2) & M64
    h ^= h >> 29
    h = (h * _P3) & M64
    h ^= h >> 32
    return h


def bloom(sids, p=0.08):
    n = len(sids)
    m = int(math.ceil(-1 * float(n) * math.log(p) / math.pow(math.log(2), 2)))
    k = int(math.ceil(math.log(2) * float(m) / float(n)))
    nbytes = 8
    while nbytes < (m + 7) // 8:
        nbytes *= 2
    bits = bytearray(nbytes)
    mask = nbytes * 8 - 1
    for sid in sids:
        key = struct.pack(">Q", sid)
        h0, h1 = xxh64(key), xxh64(key[:-1] + b"\x00")
        for i in range(k):
            loc = (h0 + h1 * i) & mask
            bits[loc >> 3] |= 1 << (loc & 7)
    return bytes(bits), m, k


def id_time(sids, rows, last_times):
    n = len(sids)
    per = 2000
    blocks = (n + per - 1) // per
    out = u32(n) + u32(blocks)
    for b in range(blocks):
        sl = slice(b * per, min(n, (b + 1) * per))
        out += u32(sl.stop - sl.start)
        for arr in ([_wrap(s) for s in sids[sl]], rows[sl], last_times[sl]):
            blk = pyenc.int_block([int(x) for x in arr])
            assert blk is not None, "the reference would use zstd here"
            out += u32(len(blk)) + blk
    return out


def build(chunks, measurement=b"mst"):
    """chunks: ascending sid, each {sid, tmin:[per seg], tmax:[per seg], times:[rows per seg], time_pages:[bytes per seg],
    columns:[(name bytes, type, [page bytes per seg], [(cells, valid) per seg])]} with columns in name order.
    Returns the file bytes."""
    out = bytearray(b"53ac2021" + u64(2))
    metas = []
    for ch in chunks:
        nseg = len(ch["time_pages"])
        chunk_off = len(out)
        cols = [(name, ty, pages, preagg(ty, [(c, v, t) for (c, v), t in zip(rows, ch["times"])]).marshal())
                for name, ty, pages, rows in ch["columns"]]
        tp = TimePreAgg()
        for t in ch["times"]:
            tp.add_values(None, None, t)
        cols.append((b"time", TYPE_INT, ch["time_pages"], tp.marshal()))
        col_meta = bytearray()
        for name, ty, pages, pre in cols:
            assert len(pages) == nseg
            out += u32(zlib.crc32(b"".join(pages)) & 0xFFFFFFFF)
            col_meta += u16(len(name)) + name + bytes([ty]) + u16(len(pre)) + pre
            for p in pages:
                col_meta += i64(len(out)) + u32(len(p))
                out += p
        meta = u64(ch["sid"]) + i64(chunk_off) + u32(len(out) - chunk_off) + u32(len(cols)) + u32(nseg)
        for a, b in zip(ch["tmin"], ch["tmax"]):
            meta += i64(a) + i64(b)
        metas.append((ch["sid"], ch["tmin"][0], ch["tmax"][-1], bytes(meta + col_meta), sum(len(t) for t in ch["times"])))
    data_end = len(out)
    index, mi, block, offs = bytearray(), [], bytearray(), []

    def close(first):
        nonlocal block, offs
        blk = bytes(block) + b"".join(u32(o) for o in offs)
        ms = metas[first:first + len(offs)]
        mi.append((ms[0][0], min(m[1] for m in ms), max(m[2] for m in ms), data_end + len(index), len(offs), len(blk)))
        index.extend(blk)
        block, offs = bytearray(), []

    first = 0
    for i, m in enumerate(metas):
        offs.append(len(block))
        block += m[3]
        if len(block) >= 256 * 1024 or len(offs) >= 512:
            close(first)
            first = i + 1
    if offs:
        close(first)
    out += index
    mi_bytes = b"".join(u64(a) + i64(b) + i64(c) + i64(d) + u32(e) + u32(f) for a, b, c, d, e, f in mi)
    out += mi_bytes
    sids = [m[0] for m in metas]
    bits, bm, bk = bloom(sids)
    out += bits
    idt = id_time(sids, [m[4] for m in metas], [m[2] for m in metas])
    out += idt
    trailer_off = len(out)
    tr = i64(16) + i64(data_end - 16) + i64(len(index)) + i64(len(mi_bytes)) + i64(len(bits)) + i64(len(idt))
    tr += i64(len(sids)) + u64(sids[0]) + u64(sids[-1]) + i64(min(m[1] for m in metas)) + i64(max(m[2] for m in metas)) + i64(len(mi)) + u64(bm) + u64(bk)
    tr += u16(8) + struct.pack("<Q", 1 | (10 << 32)) + u16(0)
    tr += u16(len(measurement)) + measurement
    out += tr + i64(trailer_off)
    return bytes(out)


# ---- a reader of every section, independent of og_tssp_parse ----
class _R:
    def __init__(self, b, p=0):
        self.b, self.p = b, p

    def take(self, n):
        v = self.b[self.p:self.p + n]
        assert len(v) == n
        self.p += n
        return v

    def u64(self):
        return struct.unpack(">Q", self.take(8))[0]

    def i64(self):
        u = self.u64()
        return (u >> 1) ^ -(u & 1)

    def u32(self):
        return struct.unpack(">I", self.take(4))[0]

    def u16(self):
        return struct.unpack(">H", self.take(2))[0]


def parse(f):
    """-> dict(trailer fields, chunks=[{sid, offset, size, tmin, tmax, columns=[{name, type, preagg, crc, segs=[(off, size)]}]}],
    meta_index=[...], bloom=bytes, id_time=bytes)."""
    assert f[:8] == b"53ac2021" and struct.unpack(">Q", f[8:16])[0] == 2
    r = _R(f, len(f) - 8)
    toff = r.i64()
    r = _R(f, toff)
    t = dict(zip(("data_off", "data_size", "index_size", "mi_size", "bloom_size", "idtime_size", "id_count"), (r.i64() for _ in range(7))))
    t["min_id"], t["max_id"] = r.u64(), r.u64()
    t["min_time"], t["max_time"], t["mi_items"] = r.i64(), r.i64(), r.i64()
    t["bloom_m"], t["bloom_k"] = r.u64(), r.u64()
    assert r.u16() == 8
    t["flags"] = struct.unpack("<Q", r.take(8))[0]
    assert r.u16() == 0
    t["name"] = r.take(r.u16())
    assert r.p == len(f) - 8
    index_off = t["data_off"] + t["data_size"]
    mi_off = index_off + t["index_size"]
    bloom_off = mi_off + t["mi_size"]
    idt_off = bloom_off + t["bloom_size"]
    assert idt_off + t["idtime_size"] == toff
    r = _R(f, mi_off)
    items, chunks = [], []
    for _ in range(t["mi_items"]):
        it = dict(id=r.u64(), tmin=r.i64(), tmax=r.i64(), off=r.i64(), count=r.u32(), size=r.u32())
        items.append(it)
        c = _R(f, it["off"])
        starts = []
        for _k in range(it["count"]):
            starts.append(c.p - it["off"])
            ch = dict(sid=c.u64(), offset=c.i64(), size=c.u32())
            ncol, nseg = c.u32(), c.u32()
            rng = [(c.i64(), c.i64()) for _s in range(nseg)]
            ch["tmin"], ch["tmax"] = [a for a, _b in rng], [b for _a, b in rng]
            ch["columns"] = []
            for _c in range(ncol):
                col = dict(name=c.take(c.u16()), type=c.take(1)[0])
                col["preagg"] = c.take(c.u16())
                col["segs"] = [(c.i64(), c.u32()) for _s in range(nseg)]
                col["crc"] = struct.unpack(">I", f[col["segs"][0][0] - 4:col["segs"][0][0]])[0]
                ch["columns"].append(col)
            chunks.append(ch)
        assert [c.u32() for _k in range(it["count"])] == starts and c.p == it["off"] + it["size"]
    return dict(trailer=t, chunks=chunks, meta_index=items, bloom=f[bloom_off:idt_off], id_time=f[idt_off:toff])
