"""Python-side handles over the libogpu C ABI (used by tests, bench.py and smoke()).

The call sequence mirrors how the reference drives this path (engine/iterators.go:130 CreateCursor ->
aggregateCursor.SinkPlan -> KeyCursor.Next, engine/comm/cursor.go:46-56):

    shard = Shard.open(...) | Shard.synth(...)       # TSSP pages + flattened ChunkMeta resident in HBM
          | Shard.open_files([(file, out_of_order), ...])  # a shard's file set, merged on the device at open
    q = AggQuery(shard, calls=[("sum", 0), ("count", 0)], interval=60e9, tmin=.., tmax=..)
    q.run()                                          # kernels
    for rec in q.records(): ...                      # Next(): ColVal-shaped views, (nil,nil,nil) == StopIteration
    d = q.dense()                                    # device-resident dense interval record (torch views, zero copy)

torch is used only as plumbing (device tensors over library-owned memory, NCCL in bench.py).
"""
import ctypes as C

import numpy as np

from . import _lib as L

_FUNCS = {"count": L.AGG_COUNT, "sum": L.AGG_SUM, "min": L.AGG_MIN, "max": L.AGG_MAX, "first": L.AGG_FIRST, "last": L.AGG_LAST}
_OPS = {"<": L.OP_LT, "<=": L.OP_LTE, ">": L.OP_GT, ">=": L.OP_GTE, "=": L.OP_EQ, "==": L.OP_EQ, "!=": L.OP_NEQ}


def _ptr(a, ctype):
    return a.ctypes.data_as(C.POINTER(ctype))


class _DevArray:
    """__cuda_array_interface__ wrapper so torch.as_tensor() can view library-owned device memory."""

    def __init__(self, ptr, n, typestr):
        self.__cuda_array_interface__ = {"shape": (n,), "typestr": typestr, "data": (int(ptr), False), "version": 2}


def device_view(ptr, n, typestr, device):
    import torch
    return torch.as_tensor(_DevArray(ptr, n, typestr), device=device)


class Shard:
    def __init__(self, handle, keepalive=None):
        self.h = C.c_void_p(handle)
        self._keep = keepalive

    @staticmethod
    def init(device=0):
        L.check(L.lib().og_init(device), "og_init")

    @staticmethod
    def desc(data, sids, series_seg_begin, seg_tmin, seg_tmax, columns, time_page_off, time_page_len):
        """An L.ShardDesc over host arrays (what Shard.open takes); the arrays it points at are kept alive as desc._keep.
        columns: list of (name, type, page_off[u64], page_len[u32]); data: bytes/np.uint8 (host)."""
        data = np.ascontiguousarray(np.frombuffer(data, dtype=np.uint8) if not isinstance(data, np.ndarray) else data)
        sids = np.ascontiguousarray(sids, dtype=np.uint64)
        ssb = np.ascontiguousarray(series_seg_begin, dtype=np.uint32)
        tmin = np.ascontiguousarray(seg_tmin, dtype=np.int64)
        tmax = np.ascontiguousarray(seg_tmax, dtype=np.int64)
        tpo = np.ascontiguousarray(time_page_off, dtype=np.uint64)
        tpl = np.ascontiguousarray(time_page_len, dtype=np.uint32)
        cds = (L.ColumnDesc * max(1, len(columns)))()
        keep = [data, sids, ssb, tmin, tmax, tpo, tpl]
        for i, (name, typ, po, pl) in enumerate(columns):
            po = np.ascontiguousarray(po, dtype=np.uint64)
            pl = np.ascontiguousarray(pl, dtype=np.uint32)
            keep += [po, pl]
            cds[i].name = name.encode()
            cds[i].type = typ
            cds[i].page_off = _ptr(po, C.c_uint64)
            cds[i].page_len = _ptr(pl, C.c_uint32)
        d = L.ShardDesc()
        d.data = _ptr(data, C.c_uint8)
        d.data_len = data.size
        d.n_series = sids.size
        d.sids = _ptr(sids, C.c_uint64)
        d.series_seg_begin = _ptr(ssb, C.c_uint32)
        d.n_segments = tmin.size
        d.seg_tmin = _ptr(tmin, C.c_int64)
        d.seg_tmax = _ptr(tmax, C.c_int64)
        d.n_columns = len(columns)
        d.columns = cds
        d.time_page_off = _ptr(tpo, C.c_uint64)
        d.time_page_len = _ptr(tpl, C.c_uint32)
        d.flags = 0
        d._keep = (keep, cds)
        return d

    @classmethod
    def open(cls, data, sids, series_seg_begin, seg_tmin, seg_tmax, columns, time_page_off, time_page_len):
        """columns: list of (name, type, page_off[u64], page_len[u32]); data: bytes/np.uint8 (host)."""
        d = cls.desc(data, sids, series_seg_begin, seg_tmin, seg_tmax, columns, time_page_off, time_page_len)
        h = C.c_void_p()
        L.check(L.lib().og_shard_open(C.byref(d), C.byref(h)), "og_shard_open")
        return cls(h.value)

    @staticmethod
    def _with_file_descs(files, call):
        """files = [(desc_or_tssp_bytes, out_of_order)] -> call(descs, flags) with every TSSP image parsed for the call's length."""
        descs = (L.ShardDesc * len(files))()
        flags = np.array([L.FILE_OUT_OF_ORDER if ooo else 0 for _f, ooo in files], dtype=np.uint32)
        keep, parsed = [], []
        try:
            for i, (f, _ooo) in enumerate(files):
                if isinstance(f, L.ShardDesc):
                    C.memmove(C.byref(descs[i]), C.byref(f), C.sizeof(L.ShardDesc))
                    continue
                buf = np.frombuffer(f, dtype=np.uint8) if not isinstance(f, np.ndarray) else np.ascontiguousarray(f, dtype=np.uint8)
                keep.append(buf)
                t = C.c_void_p()
                L.check(L.lib().og_tssp_parse(buf.ctypes.data, buf.size, C.byref(t)), "og_tssp_parse")
                parsed.append(t)
                L.check(L.lib().og_tssp_desc(t, C.byref(descs[i])), "og_tssp_desc")
            return call(descs, flags)
        finally:
            for t in parsed:
                L.lib().og_tssp_free(t)

    @classmethod
    def open_files(cls, files):
        """One shard from its ordered and out-of-order files (og_shard_open_files): files = [(desc_or_tssp_bytes, out_of_order)]
        in file-sequence order, oldest first.  A file is an L.ShardDesc (Shard.desc) or a TSSP file image, which goes through
        og_tssp_parse / og_tssp_desc.  Overlapping rows are merged on the device as the shard opens; merge_info() reports it."""
        h = C.c_void_p()

        def call(descs, flags):
            L.check(L.lib().og_shard_open_files(descs, _ptr(flags, C.c_uint32), len(files), C.byref(h)), "og_shard_open_files")
        cls._with_file_descs(files, call)
        return cls(h.value)

    def append_files(self, files):
        """Files flushed after the shard was built (og_shard_append_files), in the form open_files takes, oldest first.  The shard
        then answers as open_files over its files followed by these.  Series and column indices may move: rebuild group maps."""
        def call(descs, flags):
            L.check(L.lib().og_shard_append_files(self.h, descs, _ptr(flags, C.c_uint32), len(files)), "og_shard_append_files")
        self._with_file_descs(files, call)
        return self

    @staticmethod
    def colval(typ, values, valid, bitmap_offset=0, bitmap=True):
        """One column of a flush in the ColVal layout (lib/record/column.go): values / valid per row -> a dict of the pieces
        rows_desc takes, the non-null values packed densely, the bitmap LSB-first from bit bitmap_offset (bitmap=False: no
        bitmap, which the library accepts only when no row is null)."""
        valid = np.asarray(valid, bool)
        n = valid.size
        dt = "<u1" if typ == L.TYPE_BOOL else "<f8" if typ == L.TYPE_FLOAT else "<i8"
        dense = np.ascontiguousarray(np.asarray(values)[valid], dtype=dt)
        bm = None
        if bitmap:
            bits = np.concatenate([np.zeros(bitmap_offset, np.uint8), valid.astype(np.uint8)])
            bm = np.packbits(bits, bitorder="little") if bits.size else np.zeros(1, np.uint8)
        return dict(type=typ, val=dense.view(np.uint8), bitmap=bm, bitmap_offset=bitmap_offset, len=n, nil_count=int(n - valid.sum()))

    @staticmethod
    def rows_desc(fields, series, flags=0):
        """An L.RowsDesc (og_rows_desc) over explicit ColVal pieces.  fields: [(name, type)]; series: [(sid, times, cols)] with
        cols[f] a Shard.colval dict (its keys may be overridden) or None for a column the series lacks (len 0)."""
        keep = []
        fs = (L.RowsField * max(1, len(fields)))()
        for i, (name, typ) in enumerate(fields):
            fs[i].name, fs[i].type = name.encode(), typ
        ss = (L.RowsSeries * max(1, len(series)))()
        for k, (sid, times, cols) in enumerate(series):
            t = np.ascontiguousarray(times, dtype=np.int64)
            cv = (L.ColValView * max(1, len(fields)))()
            keep += [t, cv]
            for f, c in enumerate(cols):
                if c is None:
                    continue
                val = np.ascontiguousarray(c["val"], dtype=np.uint8)
                keep.append(val)
                cv[f].val = _ptr(val, C.c_uint8) if val.size else None
                cv[f].val_bytes = c.get("val_bytes", val.size)
                if c.get("bitmap") is not None:
                    bm = np.ascontiguousarray(c["bitmap"], dtype=np.uint8)
                    keep.append(bm)
                    cv[f].bitmap = _ptr(bm, C.c_uint8)
                cv[f].type, cv[f].len, cv[f].nil_count, cv[f].bitmap_offset = c["type"], c["len"], c["nil_count"], c["bitmap_offset"]
            ss[k].sid, ss[k].rows, ss[k].times, ss[k].cols = sid, t.size, _ptr(t, C.c_int64), cv
        d = L.RowsDesc(len(fields), fs, len(series), ss, flags)
        d._keep = (keep, fs, ss)
        return d

    @classmethod
    def batch_desc(cls, batch):
        """{sid: {"times", "cols": {name: (type, values per row, valid per row)}}} -> L.RowsDesc, fields sorted by name, a column
        a series lacks passed with len 0"""
        types = {n: t for s_ in batch.values() for n, (t, _v, _k) in s_["cols"].items()}
        names = sorted(types)
        series = [(sid, s_["times"], [cls.colval(*s_["cols"][n]) if n in s_["cols"] else None for n in names]) for sid, s_ in batch.items()]
        return cls.rows_desc([(n, types[n]) for n in names], series)

    @staticmethod
    def _rows_info(info):
        out = {k: getattr(info, k) for k, _ in L.RowsInfo._fields_ if k != "phase_ms"}
        out["phase_ms"] = list(info.phase_ms)
        return out

    def append_rows(self, batch):
        """Flush rows into the shard (og_shard_append_rows): batch is a {sid: {"times", "cols"}} dict (batch_desc) or an
        L.RowsDesc (rows_desc).  Rows are sorted and deduplicated per series, split at the series' last time in the shard into
        an ordered and an out-of-order file, encoded and appended on the device.  Returns the og_rows_info counters."""
        d = batch if isinstance(batch, L.RowsDesc) else self.batch_desc(batch)
        info = L.RowsInfo()
        L.check(L.lib().og_shard_append_rows(self.h, C.byref(d), C.byref(info)), "og_shard_append_rows")
        return self._rows_info(info)

    @classmethod
    def open_rows(cls, batch):
        """A new shard from one flush (og_shard_open_rows); batch as append_rows takes it.  The counters are sh.rows_info."""
        d = batch if isinstance(batch, L.RowsDesc) else cls.batch_desc(batch)
        info = L.RowsInfo()
        h = C.c_void_p()
        L.check(L.lib().og_shard_open_rows(C.byref(d), C.byref(h), C.byref(info)), "og_shard_open_rows")
        sh = cls(h.value)
        sh.rows_info = cls._rows_info(info)
        return sh

    def compact(self, rows_per_segment=0):
        """Re-cut every series into full segments of rows_per_segment rows (0: 1000), the last one 1..rows_per_segment, every
        column of a series with a page in each (og_shard_compact).  Returns the og_compact_info counters as a dict; all zero when
        the shard was already compact."""
        d = L.CompactDesc(rows_per_segment, 0)
        info = L.CompactInfo()
        L.check(L.lib().og_shard_compact(self.h, C.byref(d), C.byref(info)), "og_shard_compact")
        return {k: getattr(info, k) for k, _ in L.CompactInfo._fields_}

    def merge_info(self):
        m = L.MergeInfo()
        L.check(L.lib().og_shard_merge_info(self.h, C.byref(m)), "og_shard_merge_info")
        return {k: getattr(m, k) for k, _ in L.MergeInfo._fields_}

    @classmethod
    def open_desc(cls, desc, keepalive=None):
        """Open from an already-built L.ShardDesc (e.g. one produced by the oracle's host builder in tests)."""
        h = C.c_void_p()
        L.check(L.lib().og_shard_open(C.byref(desc), C.byref(h)), "og_shard_open")
        return cls(h.value, keepalive)

    @classmethod
    def open_tssp(cls, file_bytes):
        """Open a TSSP file image (bytes / numpy uint8): og_tssp_parse -> og_tssp_desc -> og_shard_open.  og_shard_open copies
        what it needs, so the parse handle is freed before returning; `measurement` and `time_range` are kept on the Shard."""
        import numpy as np
        buf = np.frombuffer(file_bytes, dtype=np.uint8) if not isinstance(file_bytes, np.ndarray) else np.ascontiguousarray(file_bytes, dtype=np.uint8)
        t = C.c_void_p()
        L.check(L.lib().og_tssp_parse(buf.ctypes.data, buf.size, C.byref(t)), "og_tssp_parse")
        try:
            d = L.ShardDesc()
            L.check(L.lib().og_tssp_desc(t, C.byref(d)), "og_tssp_desc")
            lo, hi = C.c_int64(), C.c_int64()
            L.check(L.lib().og_tssp_time_range(t, C.byref(lo), C.byref(hi)), "og_tssp_time_range")
            name = L.lib().og_tssp_measurement(t)
            columns = [(d.columns[c].name.decode(), int(d.columns[c].type)) for c in range(d.n_columns)]
            h = C.c_void_p()
            L.check(L.lib().og_shard_open(C.byref(d), C.byref(h)), "og_shard_open")
        finally:
            L.lib().og_tssp_free(t)
        sh = cls(h.value)
        sh.measurement, sh.time_range, sh.columns = name.decode(), (lo.value, hi.value), columns
        return sh

    @classmethod
    def synth(cls, n_series, rows_per_series, columns, t0=1_700_000_000_000_000_000, dt=1_000_000_000, seed=1,
              rows_per_segment=1000, series_base=0):
        """columns: list of (type, dist, null_permille). Builds the shard on the device with the encode kernels."""
        cols = (L.SynthColumn * len(columns))()
        for i, (t, dist, npm) in enumerate(columns):
            cols[i].type, cols[i].dist, cols[i].null_permille = t, dist, npm
        d = L.SynthDesc(n_series, rows_per_series, rows_per_segment, t0, dt, seed, len(columns), cols, series_base)
        h = C.c_void_p()
        L.check(L.lib().og_shard_synth(C.byref(d), C.byref(h)), "og_shard_synth")
        return cls(h.value)

    def info(self):
        a = [C.c_uint64() for _ in range(4)]
        t = [C.c_int64(), C.c_int64()]
        L.check(L.lib().og_shard_info(self.h, *[C.byref(x) for x in a], C.byref(t[0]), C.byref(t[1])), "og_shard_info")
        return dict(n_series=a[0].value, n_segments=a[1].value, n_rows=a[2].value, page_bytes=a[3].value, tmin=t[0].value, tmax=t[1].value)

    def export(self):
        lay = L.ShardLayout()
        L.check(L.lib().og_shard_layout_get(self.h, C.byref(lay)), "og_shard_layout_get")
        ns, ng, nc = lay.n_series, lay.n_segments, lay.n_columns
        out = dict(data=np.empty(lay.data_len, np.uint8), sids=np.empty(ns, np.uint64), series_seg_begin=np.empty(ns + 1, np.uint32),
                   seg_tmin=np.empty(ng, np.int64), seg_tmax=np.empty(ng, np.int64), page_off=np.empty((nc + 1, ng), np.uint64),
                   page_len=np.empty((nc + 1, ng), np.uint32), col_types=np.empty(nc, np.int32))
        L.check(L.lib().og_shard_export(self.h, *[out[k].ctypes.data for k in
                                                   ("data", "sids", "series_seg_begin", "seg_tmin", "seg_tmax", "page_off", "page_len", "col_types")]),
                "og_shard_export")
        return out

    def downsample(self, column, interval, tmin, tmax):
        """og_downsample: per-series min/max/sum/count/first/last of `column` per window -> re-encoded pages, in one library call
        (the pass downsample_shard runs, with those six calls on one float or int field)."""
        h = C.c_void_p()
        L.check(L.lib().og_downsample(self.h, column, interval, tmin, tmax, C.byref(h)), "og_downsample")
        return Downsampled(h.value)

    def downsample_shard(self, interval, tmin, tmax, ops):
        """og_downsample_shard: every field under a per-type call list -> <call>_<field> columns with null cells, in one library
        call.  ops: {OG type: [call name or OG_AGG_* value, ...]}; a type without an entry drops its fields."""
        entries = list(ops.items())
        arr = (L.DownsampleOps * max(1, len(entries)))()
        keep = []
        for i, (typ, funcs) in enumerate(entries):
            f = (C.c_int32 * max(1, len(funcs)))(*[_FUNCS[x] if isinstance(x, str) else int(x) for x in funcs])
            keep.append(f)
            arr[i].type, arr[i].n_funcs, arr[i].funcs = int(typ), len(funcs), C.cast(f, L.i32p)
        d = L.DownsampleDesc(int(interval), int(tmin), int(tmax), len(entries), arr)
        h = C.c_void_p()
        L.check(L.lib().og_downsample_shard(self.h, C.byref(d), C.byref(h)), "og_downsample_shard")
        return Downsampled(h.value)

    def decode_segment(self, seg, descending=False):
        rv = L.RecordView()
        L.check(L.lib().og_decode_segment_ex(self.h, seg, 1 if descending else 0, C.byref(rv)), "og_decode_segment_ex")
        return _record_to_py(rv)

    def close(self):
        if self.h:
            L.lib().og_shard_close(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def write_tssp(shard, measurement, series=None, timing=None):
    """og_shard_write_tssp: the bytes of one TSSP file holding `shard` (any open Shard: from a description or file, synthesised,
    merged, or a downsample result reopened with Downsampled.open()).  series: (begin, end) half-open range of the shard's series,
    None = all.  timing: a dict that receives the milliseconds of the call's phases."""
    d = L.TsspWriteDesc(measurement.encode() if isinstance(measurement, str) else measurement, *((0, 0) if series is None else series), 0)
    h = C.c_void_p()
    L.check(L.lib().og_shard_write_tssp(shard.h, C.byref(d), C.byref(h)), "og_shard_write_tssp")
    try:
        n = C.c_uint64()
        L.check(L.lib().og_tssp_image_size(h, C.byref(n)), "og_tssp_image_size")
        out = np.empty(n.value, np.uint8)
        L.check(L.lib().og_tssp_image_export(h, out.ctypes.data), "og_tssp_image_export")
        if timing is not None:
            ms = (C.c_double * 4)()
            L.check(L.lib().og_tssp_image_timing(h, ms), "og_tssp_image_timing")
            timing.update(preagg=ms[0], layout_gather_crc=ms[1], metadata_d2h=ms[2], host_assembly=ms[3])
    finally:
        L.lib().og_tssp_image_free(h)
    return out.tobytes()


class Downsampled:
    """Result of Shard.downsample or Shard.downsample_shard: a shard description whose pages live in device memory (owned by this handle)."""

    def __init__(self, h):
        self.h = h
        self.desc = L.ShardDesc()
        rows = C.c_uint64()
        L.check(L.lib().og_downsampled_desc(self.h, C.byref(self.desc), C.byref(rows)), "og_downsampled_desc")
        self.rows = rows.value

    def open(self):
        """Open the new shard in place (zero-copy: OG_SHARD_DEVICE_DATA); this object must outlive the returned Shard."""
        return Shard.open_desc(self.desc, keepalive=self)

    def export(self):
        out = np.empty(max(1, self.desc.data_len), np.uint8)
        L.check(L.lib().og_downsampled_export(self.h, out.ctypes.data), "og_downsampled_export")
        return out[:self.desc.data_len]

    def timing(self):
        """Milliseconds of the downsample pass's phases."""
        ms = (C.c_double * 4)()
        L.check(L.lib().og_downsampled_timing(self.h, ms), "og_downsampled_timing")
        return dict(queries=ms[0], keep_scatter=ms[1], encode=ms[2], assembly=ms[3])

    def columns(self):
        """[(name, type, page_off, page_len)] of the field columns, then the time column's (page_off, page_len)."""
        d, ng = self.desc, self.desc.n_segments
        cols = [(d.columns[c].name.decode(), int(d.columns[c].type),
                 np.ctypeslib.as_array(d.columns[c].page_off, shape=(ng,)).copy() if ng else np.empty(0, np.uint64),
                 np.ctypeslib.as_array(d.columns[c].page_len, shape=(ng,)).copy() if ng else np.empty(0, np.uint32))
                for c in range(d.n_columns)]
        t = (np.ctypeslib.as_array(d.time_page_off, shape=(ng,)).copy() if ng else np.empty(0, np.uint64),
             np.ctypeslib.as_array(d.time_page_len, shape=(ng,)).copy() if ng else np.empty(0, np.uint32))
        return cols, t

    def close(self):
        if self.h:
            L.lib().og_downsampled_free(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def _record_to_py(rv):
    cols = []
    for i in range(rv.n_cols):
        cv = rv.cols[i]
        raw = np.ctypeslib.as_array(cv.val, shape=(cv.val_bytes,)).copy() if cv.val_bytes else np.empty(0, np.uint8)
        if cv.type == L.TYPE_FLOAT:
            vals = raw.view(np.float64)
        elif cv.type == L.TYPE_INT:
            vals = raw.view(np.int64)
        else:
            vals = raw
        nb = (cv.bitmap_offset + cv.len + 7) // 8
        bm = np.ctypeslib.as_array(cv.bitmap, shape=(nb,)).copy() if nb else np.empty(0, np.uint8)
        valid = np.unpackbits(bm, bitorder="little")[cv.bitmap_offset:cv.bitmap_offset + cv.len].astype(bool)
        times = np.ctypeslib.as_array(cv.times, shape=(cv.len,)).copy() if cv.times else None
        cols.append(dict(type=cv.type, values=vals, valid=valid, len=cv.len, nil_count=cv.nil_count, times=times))
    times = np.ctypeslib.as_array(rv.times, shape=(rv.rows,)).copy() if rv.rows else np.empty(0, np.int64)
    return dict(cols=cols, times=times, rows=rv.rows, group=rv.group, sid=rv.sid)


class ScanCursor:
    """Record materialisation for non-aggregating callers: the KeyCursor.Next() of a plain scan (what HybridStoreReader drains,
    engine/hybrid_store_reader.go:444; per file it is Location.readData, engine/immutable/location.go:261-330: segments of a
    chunk in time order — reversed for descending scans — pruned by ChunkMeta.timeRange, decoded by decodeColumnData
    reader.go:674 and cut to the query range by FilterByTime reader.go:754).

    One record per qualifying segment: series in shard order, a series' segments oldest first (latest first when
    ascending=False, with the rows of each record reversed by the device: og_decode_segment_ex OG_DECODE_DESCENDING).  Rows
    outside [tmin, tmax] are dropped; a column's `values` stay dense over its non-null rows, like ColVal.Val."""

    def __init__(self, shard, tmin, tmax, ascending=True):
        self.shard, self.tmin, self.tmax, self.ascending = shard, tmin, tmax, ascending
        lay = L.ShardLayout()
        L.check(L.lib().og_shard_layout_get(shard.h, C.byref(lay)), "og_shard_layout_get")
        ns, ng = lay.n_series, lay.n_segments
        self.sids, self.ssb = np.empty(ns, np.uint64), np.empty(ns + 1, np.uint32)
        self.seg_tmin, self.seg_tmax = np.empty(ng, np.int64), np.empty(ng, np.int64)
        L.check(L.lib().og_shard_export(shard.h, None, self.sids.ctypes.data, self.ssb.ctypes.data, self.seg_tmin.ctypes.data,
                                        self.seg_tmax.ctypes.data, None, None, None), "og_shard_export")

    def segments(self):
        """(series index, segment) in emission order, after time-range pruning (location.go:276-280)."""
        for s in range(self.sids.size):
            segs = range(int(self.ssb[s]), int(self.ssb[s + 1]))
            for g in (segs if self.ascending else reversed(segs)):
                if self.seg_tmax[g] >= self.tmin and self.seg_tmin[g] <= self.tmax:
                    yield s, g

    def __iter__(self):
        for s, g in self.segments():
            rec = self.shard.decode_segment(g, descending=not self.ascending)
            t = rec["times"]
            keep = (t >= self.tmin) & (t <= self.tmax)
            if not keep.all():
                if not keep.any():
                    continue
                for c in rec["cols"]:
                    dense_keep = keep[c["valid"]]  # the kept rows among the non-null ones
                    c["values"] = c["values"][dense_keep]
                    c["valid"] = c["valid"][keep]
                    c["len"] = int(keep.sum())
                    c["nil_count"] = int(c["len"] - c["valid"].sum())
                rec["times"] = t[keep]
                rec["rows"] = int(keep.sum())
            rec["sid"] = int(self.sids[s])
            rec["segment"] = g
            yield rec


class AggQuery:
    """calls: list of (func_name, column); filter: RPN list of ("term", column, op, const) | "and" | "or"."""

    def __init__(self, shard, calls, interval, tmin, tmax, offset=0, filter=None, group="all", series_group=None,
                 n_groups=0, chunk_size=1024, flags=0, ascending=True):
        self.shard = shard
        self._calls = (L.Call * len(calls))()
        for i, (f, c) in enumerate(calls):
            self._calls[i].func = _FUNCS[f] if isinstance(f, str) else f
            self._calls[i].column = c
        flt = filter or []
        self._filter = (L.FilterItem * max(1, len(flt)))()
        for i, it in enumerate(flt):
            if it in ("and", "or"):
                self._filter[i].kind = L.F_AND if it == "and" else L.F_OR
            else:
                _, col, op, const = it
                self._filter[i].kind = L.F_TERM
                self._filter[i].column = col
                self._filter[i].op = _OPS[op]
                if isinstance(const, float):
                    self._filter[i].const_is_float, self._filter[i].fval = 1, const
                else:
                    self._filter[i].const_is_float, self._filter[i].ival = 0, int(const)
        d = L.QueryDesc()
        d.interval, d.offset, d.tmin, d.tmax, d.ascending = int(interval), int(offset), int(tmin), int(tmax), 1 if ascending else 0
        d.n_calls, d.calls = len(calls), self._calls
        d.n_filter, d.filter = len(flt), self._filter
        d.group_mode = {"all": L.GROUP_ALL, "series": L.GROUP_PER_SERIES, "map": L.GROUP_MAP}[group]
        self._sg = None
        if group == "map":
            self._sg = np.ascontiguousarray(series_group, dtype=np.uint32)
            d.series_group, d.n_groups = _ptr(self._sg, C.c_uint32), int(n_groups)
        d.chunk_size, d.flags = chunk_size, flags
        self.desc = d
        self.h = C.c_void_p()
        L.check(L.lib().og_query_create(shard.h, C.byref(d), C.byref(self.h)), "og_query_create")

    def run(self):
        L.check(L.lib().og_query_run(self.h), "og_query_run")
        return self

    def stats(self):
        s = L.Stats()
        L.check(L.lib().og_query_stats(self.h, C.byref(s)), "og_query_stats")
        return {k: getattr(s, k) for k, _ in L.Stats._fields_}

    def dense_view(self):
        dv = L.DenseView()
        L.check(L.lib().og_query_dense(self.h, C.byref(dv)), "og_query_dense")
        return dv

    def dense(self, device=None):
        """Zero-copy torch views of the dense interval record: list of dict(values, valid, times|None, type, func)."""
        import torch
        dv = self.dense_view()
        device = device or torch.device("cuda", torch.cuda.current_device())
        n = dv.n_groups * dv.n_buckets
        cols = []
        for i in range(dv.n_cols):
            c = dv.cols[i]
            vals = device_view(c.values, n, "<f8" if c.type == L.TYPE_FLOAT else "<i8", device)
            valid = device_view(c.valid, n, "|u1", device)
            times = device_view(c.times, n, "<i8", device) if c.times else None
            cols.append(dict(values=vals, valid=valid, times=times, type=c.type, func=c.func))
        return dict(n_groups=dv.n_groups, n_buckets=dv.n_buckets, start=dv.start, interval=dv.interval, cols=cols)

    def dense_host(self):
        d = self.dense()
        for c in d["cols"]:
            c["values"] = c["values"].cpu().numpy()
            c["valid"] = c["valid"].cpu().numpy()
            c["times"] = c["times"].cpu().numpy() if c["times"] is not None else None
        return d

    def records(self):
        rv = L.RecordView()
        while True:
            st = L.lib().og_query_next(self.h, C.byref(rv))
            if st == L.OG_EOF:
                return
            L.check(st, "og_query_next")
            yield _record_to_py(rv)

    def abort(self):
        L.lib().og_query_abort(self.h)

    def close(self):
        if self.h:
            L.lib().og_query_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class Comm:
    """The library's own NCCL communicator (og_comm_*): rank 0 creates the 128-byte id, the host passes it to the other
    ranks through whatever channel it has (a Go host: its RPC layer; bench.py: torch.distributed's store), every rank
    then joins.  allreduce(q) merges q's dense interval record over all ranks in place (og_query_allreduce)."""

    def __init__(self, handle, rank, world):
        self.h, self.rank, self.world = handle, rank, world

    @staticmethod
    def _prefer_bundled_nccl():
        """libogpu dlopens "libnccl.so.2".  When PyTorch is installed it ships its own copy under the same SONAME; whichever is
        loaded first serves the whole process, and an older system copy loaded first breaks a later `import torch`.  Point
        OGPU_NCCL_LIB at the bundled one (no torch import needed) unless the caller chose a library."""
        import importlib.util
        import os
        if os.environ.get("OGPU_NCCL_LIB"):
            return
        spec = importlib.util.find_spec("nvidia.nccl") if importlib.util.find_spec("nvidia") else None
        for base in (list(spec.submodule_search_locations) if spec and spec.submodule_search_locations else []):
            cand = os.path.join(base, "lib", "libnccl.so.2")
            if os.path.exists(cand):
                os.environ["OGPU_NCCL_LIB"] = cand
                return

    @staticmethod
    def unique_id():
        Comm._prefer_bundled_nccl()
        buf = (C.c_uint8 * 128)()
        L.check(L.lib().og_comm_unique_id(buf), "og_comm_unique_id")
        return bytes(buf)

    @classmethod
    def init_rank(cls, uid, rank, world):
        cls._prefer_bundled_nccl()
        buf = (C.c_uint8 * 128).from_buffer_copy(uid)
        h = C.c_void_p()
        L.check(L.lib().og_comm_init_rank(buf, int(rank), int(world), C.byref(h)), "og_comm_init_rank")
        return cls(h, rank, world)

    def info(self):
        r, w, v = C.c_int(), C.c_int(), C.c_int()
        L.check(L.lib().og_comm_info(self.h, C.byref(r), C.byref(w), C.byref(v)), "og_comm_info")
        return dict(rank=r.value, world=w.value, nccl_version=v.value)

    def allreduce_f64(self, vals, op="sum"):
        arr = (C.c_double * len(vals))(*vals)
        L.check(L.lib().og_comm_allreduce_f64(self.h, arr, len(vals), 1 if op == "max" else 0), "og_comm_allreduce_f64")
        return list(arr)

    def allreduce(self, query):
        L.check(L.lib().og_query_allreduce(query.h, self.h), "og_query_allreduce")

    def close(self):
        if self.h:
            L.lib().og_comm_destroy(self.h)
            self.h = None

