"""Downsample a shard on the device: decode + per-series re-aggregation to coarser buckets + re-encode to TSSP pages
(SURVEY §8f row 3, configs[4] shape).

Reference path this stands for: engine/record_plan.go:494-830 (FileSequenceAggregator pulls records, newProcessor reduces them per
series) feeding engine/immutable/stream_downsample.go:454-600 (re-encode the downsampled columns with the ordinary column builders).
Both functions here are one library call each, and both run the same pass (csrc/downsample.cu): the read-aggregate half is the
same C-ABI query as everywhere else (OG_GROUP_PER_SERIES), the write half is the device page encoder.

downsample() is one numeric field with the reference's downsample schema (og_downsample): min_, max_, sum_, count_, first_, last_
of the source field, window start as the row time, empty windows dropped (lib/record/record.go:1298-1365 TransIntervalRec2Rec).
downsample_shard() is the whole shard (og_downsample_shard): every field under the policy's call list for its type,
<call>_<field> columns, null cells where a field had no value in a kept window.

No CPU fallback: every step runs through libogpu.so.
"""
import ctypes as C

import numpy as np

from .cursor import device_view

OUT_CALLS = ("min", "max", "sum", "count", "first", "last")


def _result(ds):
    """The dict both functions return, from a Downsampled handle (which the caller still closes)."""
    import torch

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


def downsample(shard, column, interval, tmin, tmax):
    """One float or int field in one library call (og_downsample): per series and window, min/max/sum/count/first/last of
    `column`, named <call>_f<column> in that order.  Returns dict(data=uint8 torch tensor on the device, with the 1024-byte
    tail readers need, data_len, columns=[(name, type, page_off, page_len)], names, time_page_off, time_page_len,
    series_seg_begin, seg_tmin, seg_tmax, sids, rows=int, timing={phase: ms}) describing a new shard whose fields are the six
    aggregates."""
    ds = shard.downsample(column, interval, tmin, tmax)
    try:
        return _result(ds)
    finally:
        ds.close()


def downsample_shard(shard, interval, tmin, tmax, ops):
    """Every field of `shard` under a per-type policy in one library call (og_downsample_shard): ops = {OG type: [call, ...]},
    e.g. {L.TYPE_FLOAT: ["min", "max", "sum", "count", "first", "last"], L.TYPE_BOOL: ["count", "last"]}.  Fields of a type
    without an entry are dropped; each output column is named <call>_<field>; a series keeps a window where any of its
    output cells is non-null, and cells without a value are null (their pages carry a bitmap).

    Returns the dict downsample() returns."""
    ds = shard.downsample_shard(interval, tmin, tmax, ops)
    try:
        return _result(ds)
    finally:
        ds.close()
