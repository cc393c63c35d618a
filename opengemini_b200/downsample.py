"""Downsample a shard on the device: decode + per-series re-aggregation to coarser buckets + re-encode to TSSP pages
(SURVEY §8f row 3, configs[4] shape).

Reference path this stands for: engine/record_plan.go:494-830 (FileSequenceAggregator pulls records, newProcessor reduces them per
series) feeding engine/immutable/stream_downsample.go:454-600 (re-encode the downsampled columns with the ordinary column builders).
Here the read-aggregate half is the same C-ABI query as everywhere else (OG_GROUP_PER_SERIES), the write half is og_encode_pages;
torch is only used to reshape device arrays between the two calls.  Output column set and naming follow the reference's
downsample schema: min_, max_, sum_, count_, first_, last_ of the source field, window start as the row time, empty windows
dropped (lib/record/record.go:1298-1365 TransIntervalRec2Rec).

downsample_shard() is the whole-shard form behind one library call (og_downsample_shard): every field under the policy's call list
for its type, <call>_<field> columns, null cells where a field had no value in a kept window.

No CPU fallback: every step runs through libogpu.so.
"""
import ctypes as C

import numpy as np

from . import _lib as L
from .cursor import AggQuery, device_view

OUT_CALLS = ("min", "max", "sum", "count", "first", "last")
ROWS_PER_SEGMENT = 1000  # lib/util/util.go:72


def downsample(shard, column, interval, tmin, tmax, col_type=L.TYPE_FLOAT):
    """Returns dict(data=uint8 torch tensor on the device, columns=[(name, type, page_off, page_len)], time_page_off, time_page_len,
    series_seg_begin, seg_tmin, seg_tmax, sids, rows=int) describing a new shard whose fields are the six aggregates."""
    import torch

    q = AggQuery(shard, [(f, column) for f in OUT_CALLS], interval, tmin, tmax, group="series").run()
    try:
        d = q.dense()
        ns, nb = d["n_groups"], d["n_buckets"]
        dev = d["cols"][0]["values"].device
        keep = d["cols"][3]["valid"].view(ns, nb).bool()  # count > 0 <=> the window has rows (all six share it)
        rows_s = keep.sum(1)  # rows per series after dropping empty windows
        # stable partition of every series row: kept buckets first, in time order
        order = torch.argsort((~keep).to(torch.uint8), dim=1, stable=True)
        segs_s = (rows_s + ROWS_PER_SEGMENT - 1) // ROWS_PER_SEGMENT
        max_segs = max(1, (nb + ROWS_PER_SEGMENT - 1) // ROWS_PER_SEGMENT)
        pad = max_segs * ROWS_PER_SEGMENT
        g = torch.arange(max_segs, device=dev).view(1, max_segs)
        seg_rows = (rows_s.view(ns, 1) - g * ROWS_PER_SEGMENT).clamp(0, ROWS_PER_SEGMENT)  # [ns, max_segs]
        live = seg_rows > 0
        seg_rows_live = seg_rows[live].to(torch.int32).contiguous()
        n_seg = int(seg_rows_live.numel())
        win_start = d["start"] + torch.arange(nb, device=dev, dtype=torch.int64) * d["interval"]

        def to_segments(x2d):
            """[ns, nb] -> kept entries first -> padded to whole segments -> only the non-empty segments, [n_seg, 1000]."""
            x = torch.gather(x2d, 1, order)
            if pad > nb:
                x = torch.nn.functional.pad(x, (0, pad - nb))
            return x.view(ns, max_segs, ROWS_PER_SEGMENT)[live].contiguous()

        lib = L.lib()
        blobs, columns, pos = [], [], 0

        def encode(typ, is_time, seg_vals):
            nonlocal pos
            cap = n_seg * 8800
            out = torch.empty(cap, dtype=torch.uint8, device=dev)
            off = torch.empty(n_seg, dtype=torch.int64, device=dev)
            ln = torch.empty(n_seg, dtype=torch.int32, device=dev)
            total = C.c_uint64()
            L.check(lib.og_encode_pages(typ, is_time, seg_vals.data_ptr(), None, seg_rows_live.data_ptr(), n_seg, ROWS_PER_SEGMENT,
                                        out.data_ptr(), cap, off.data_ptr(), ln.data_ptr(), C.byref(total)), "og_encode_pages")
            blobs.append(out[: total.value])
            po = (off + pos).cpu().numpy().astype(np.uint64)
            pos += int(total.value)
            return po, ln.cpu().numpy().astype(np.uint32)

        for k, f in enumerate(OUT_CALLS):
            c = d["cols"][k]
            typ = L.TYPE_INT if f == "count" else col_type
            vals = c["values"].view(torch.int64).view(ns, nb)  # raw 8-byte cells
            po, pl = encode(typ, 0, to_segments(vals))
            columns.append((f"{f}_f{column}", typ, po, pl))
        t_seg = to_segments(win_start.view(1, nb).expand(ns, nb).contiguous())
        tpo, tpl = encode(L.TYPE_INT, 1, t_seg)
        rows_live = seg_rows_live.to(torch.int64)
        seg_tmin = t_seg[:, 0].cpu().numpy()
        seg_tmax = torch.gather(t_seg, 1, (rows_live - 1).view(-1, 1)).view(-1).cpu().numpy()
        ssb = np.concatenate([[0], np.cumsum(segs_s.cpu().numpy())]).astype(np.uint32)
        data = torch.cat(blobs + [torch.zeros(1024, dtype=torch.uint8, device=dev)])
        return dict(data=data, data_len=pos, columns=columns, time_page_off=tpo, time_page_len=tpl, series_seg_begin=ssb,
                    seg_tmin=seg_tmin, seg_tmax=seg_tmax, sids=np.arange(1, ns + 1, dtype=np.uint64), rows=int(rows_s.sum()))
    finally:
        q.close()


def downsample_shard(shard, interval, tmin, tmax, ops):
    """Every field of `shard` under a per-type policy in one library call (og_downsample_shard): ops = {OG type: [call, ...]},
    e.g. {L.TYPE_FLOAT: ["min", "max", "sum", "count", "first", "last"], L.TYPE_BOOL: ["count", "last"]}.  Fields of a type
    without an entry are dropped; each output column is named <call>_<field>; a series keeps a window where any of its
    output cells is non-null, and cells without a value are null (their pages carry a bitmap).

    Returns the dict downsample() returns (data: uint8 torch tensor on the device, with the 1024-byte tail readers need), plus
    names=[column names in schema order] and timing={phase: ms}."""
    import torch

    ds = shard.downsample_shard(interval, tmin, tmax, ops)
    try:
        d = ds.desc
        columns, (tpo, tpl) = ds.columns()
        ns, ng = d.n_series, d.n_segments
        dev = torch.device("cuda", torch.cuda.current_device())
        # the handle owns the pages: copy them (device to device) into a tensor that outlives it
        data = device_view(C.cast(d.data, C.c_void_p).value, d.data_len + 1024, "|u1", dev).clone()
        torch.cuda.synchronize(dev)
        return dict(data=data, data_len=int(d.data_len), columns=columns, names=[c[0] for c in columns], time_page_off=tpo,
                    time_page_len=tpl, series_seg_begin=np.ctypeslib.as_array(d.series_seg_begin, shape=(ns + 1,)).copy(),
                    seg_tmin=np.ctypeslib.as_array(d.seg_tmin, shape=(ng,)).copy() if ng else np.empty(0, np.int64),
                    seg_tmax=np.ctypeslib.as_array(d.seg_tmax, shape=(ng,)).copy() if ng else np.empty(0, np.int64),
                    sids=np.ctypeslib.as_array(d.sids, shape=(ns,)).copy() if ns else np.empty(0, np.uint64), rows=int(ds.rows),
                    timing=ds.timing())
    finally:
        ds.close()
