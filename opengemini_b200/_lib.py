"""ctypes binding of libogpu.so (include/ogpu.h).

The library is the product; this module only marshals arguments.  It fails loudly when the
CUDA library is missing — there is no Python/CPU fallback for any compute entry point.
"""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("OGPU_LIB") or os.path.join(_HERE, "libogpu.so")  # OGPU_LIB: A/B builds of the same library (tools/)

# ---- status codes / enums (mirror include/ogpu.h) ----
OG_OK, OG_EOF = 0, 1
OG_E_INVAL, OG_E_CUDA, OG_E_NOMEM, OG_E_UNSUPPORTED, OG_E_CORRUPT, OG_E_ABORTED, OG_E_TYPE, OG_E_STATE = -1, -2, -3, -4, -5, -6, -7, -8
TYPE_INT, TYPE_FLOAT, TYPE_STRING, TYPE_BOOL = 1, 3, 4, 5
AGG_COUNT, AGG_SUM, AGG_MIN, AGG_MAX, AGG_FIRST, AGG_LAST = 1, 2, 3, 4, 5, 6
F_TERM, F_AND, F_OR = 0, 1, 2
OP_LT, OP_LTE, OP_GT, OP_GTE, OP_EQ, OP_NEQ = 0, 1, 2, 3, 4, 5
GROUP_ALL, GROUP_PER_SERIES, GROUP_MAP = 0, 1, 2
Q_STRICT_ORDER = 1
Q_NO_FUSED = 2
Q_NO_FAST = 4
Q_QUERY_GRID = 16
SYNTH_F_HI, SYNTH_F_LO, SYNTH_INT_WALK, SYNTH_BOOL = 0, 1, 2, 3
SHARD_DEVICE_DATA = 1
FILE_OUT_OF_ORDER = 1

u8p, u32p, u64p, i64p, i32p = C.POINTER(C.c_uint8), C.POINTER(C.c_uint32), C.POINTER(C.c_uint64), C.POINTER(C.c_int64), C.POINTER(C.c_int32)


class FilterItem(C.Structure):
    _fields_ = [("kind", C.c_int32), ("column", C.c_int32), ("op", C.c_int32), ("const_is_float", C.c_int32),
                ("fval", C.c_double), ("ival", C.c_int64)]


class Call(C.Structure):
    _fields_ = [("func", C.c_int32), ("column", C.c_int32)]


class QueryDesc(C.Structure):
    _fields_ = [("interval", C.c_int64), ("offset", C.c_int64), ("tmin", C.c_int64), ("tmax", C.c_int64),
                ("ascending", C.c_int32), ("n_calls", C.c_uint32), ("calls", C.POINTER(Call)),
                ("n_filter", C.c_uint32), ("filter", C.POINTER(FilterItem)), ("group_mode", C.c_int32),
                ("n_groups", C.c_uint32), ("series_group", u32p), ("chunk_size", C.c_int32), ("flags", C.c_uint32)]


class ColumnDesc(C.Structure):
    _fields_ = [("name", C.c_char_p), ("type", C.c_int32), ("page_off", u64p), ("page_len", u32p)]


class ShardDesc(C.Structure):
    _fields_ = [("data", u8p), ("data_len", C.c_uint64), ("n_series", C.c_uint32), ("sids", u64p),
                ("series_seg_begin", u32p), ("n_segments", C.c_uint32), ("seg_tmin", i64p), ("seg_tmax", i64p),
                ("n_columns", C.c_uint32), ("columns", C.POINTER(ColumnDesc)), ("time_page_off", u64p),
                ("time_page_len", u32p), ("flags", C.c_uint32)]


class ColValView(C.Structure):
    _fields_ = [("val", u8p), ("val_bytes", C.c_uint64), ("bitmap", u8p), ("times", i64p), ("type", C.c_int32),
                ("len", C.c_int32), ("nil_count", C.c_int32), ("bitmap_offset", C.c_int32)]


class RecordView(C.Structure):
    _fields_ = [("n_cols", C.c_uint32), ("cols", C.POINTER(ColValView)), ("times", i64p), ("rows", C.c_int32),
                ("group", C.c_uint32), ("sid", C.c_uint64)]


class DenseCol(C.Structure):
    _fields_ = [("values", C.c_void_p), ("valid", C.c_void_p), ("times", C.c_void_p), ("type", C.c_int32), ("func", C.c_int32)]


class DenseView(C.Structure):
    _fields_ = [("n_groups", C.c_uint32), ("n_buckets", C.c_uint32), ("start", C.c_int64), ("interval", C.c_int64),
                ("n_cols", C.c_uint32), ("cols", C.POINTER(DenseCol)), ("stream", C.c_void_p)]


class Stats(C.Structure):
    _fields_ = [("rows_decoded", C.c_uint64), ("segments_scanned", C.c_uint64), ("page_bytes", C.c_uint64),
                ("dir_bytes", C.c_uint64), ("out_bytes", C.c_uint64), ("kernel_ms", C.c_double), ("h2d_ms", C.c_double), ("main_kernel_ms", C.c_double),
                ("kernel_launches", C.c_uint32), ("path", C.c_int32), ("il_state", C.c_int32), ("per_series_cells_used", C.c_int32),
                ("il_build_ms", C.c_double), ("il_bytes", C.c_uint64), ("general_segments", C.c_uint64), ("merge_ms", C.c_double),
                ("il_packed_segments", C.c_uint64)]


class SynthColumn(C.Structure):
    _fields_ = [("type", C.c_int32), ("dist", C.c_int32), ("null_permille", C.c_uint32)]


class SynthDesc(C.Structure):
    _fields_ = [("n_series", C.c_uint32), ("rows_per_series", C.c_uint32), ("rows_per_segment", C.c_uint32),
                ("t0", C.c_int64), ("dt", C.c_int64), ("seed", C.c_uint64), ("n_columns", C.c_uint32),
                ("columns", C.POINTER(SynthColumn)), ("series_base", C.c_uint32)]


class ShardLayout(C.Structure):
    _fields_ = [("data_len", C.c_uint64), ("n_series", C.c_uint32), ("n_segments", C.c_uint32), ("n_columns", C.c_uint32)]


class DownsampleOps(C.Structure):
    _fields_ = [("type", C.c_int32), ("n_funcs", C.c_uint32), ("funcs", i32p)]


class DownsampleDesc(C.Structure):
    _fields_ = [("interval", C.c_int64), ("tmin", C.c_int64), ("tmax", C.c_int64), ("n_types", C.c_uint32),
                ("ops", C.POINTER(DownsampleOps))]


class MergeInfo(C.Structure):
    _fields_ = [("n_files", C.c_uint32), ("n_out_of_order_files", C.c_uint32), ("series_merged", C.c_uint64),
                ("out_of_order_rows", C.c_uint64), ("rows_replaced", C.c_uint64), ("rows_after_merge", C.c_uint64),
                ("segments_kept", C.c_uint64), ("segments_rewritten_in", C.c_uint64), ("segments_rewritten_out", C.c_uint64),
                ("merge_ms", C.c_double)]


class CompactDesc(C.Structure):
    _fields_ = [("rows_per_segment", C.c_uint32), ("flags", C.c_uint32)]


class CompactInfo(C.Structure):
    _fields_ = [("series_rewritten", C.c_uint64), ("segments_kept", C.c_uint64), ("segments_rewritten_in", C.c_uint64),
                ("segments_rewritten_out", C.c_uint64), ("rows_rewritten", C.c_uint64), ("compact_ms", C.c_double)]


class RowsField(C.Structure):
    _fields_ = [("name", C.c_char_p), ("type", C.c_int32)]


class RowsSeries(C.Structure):
    _fields_ = [("sid", C.c_uint64), ("rows", C.c_uint32), ("times", i64p), ("cols", C.POINTER(ColValView))]


class RowsDesc(C.Structure):
    _fields_ = [("n_fields", C.c_uint32), ("fields", C.POINTER(RowsField)), ("n_series", C.c_uint32),
                ("series", C.POINTER(RowsSeries)), ("flags", C.c_uint32)]


class RowsInfo(C.Structure):
    _fields_ = [("series_in", C.c_uint64), ("rows_in", C.c_uint64), ("rows_replaced", C.c_uint64), ("ordered_rows", C.c_uint64),
                ("out_of_order_rows", C.c_uint64), ("segments_written", C.c_uint64), ("phase_ms", C.c_double * 4)]


class TsspWriteDesc(C.Structure):
    _fields_ = [("measurement", C.c_char_p), ("series_begin", C.c_uint32), ("series_end", C.c_uint32), ("flags", C.c_uint32)]


# every symbol include/ogpu.h declares (checked by tests/test_abi.py against the header text)
EXPORTS = [
    "og_init", "og_device_count", "og_strerror", "og_last_error", "og_version", "og_shard_open", "og_shard_close",
    "og_shard_info", "og_query_create", "og_query_run", "og_query_next", "og_query_dense", "og_query_stats",
    "og_query_abort", "og_query_destroy", "og_query_merge_dense", "og_decode_segment", "og_decode_segment_ex", "og_decode_column_device",
    "og_shard_synth", "og_shard_layout_get", "og_shard_export", "og_encode_pages",
    "og_release_cached_memory", "og_comm_unique_id", "og_comm_init_rank", "og_comm_destroy", "og_comm_info", "og_comm_allreduce_f64", "og_query_allreduce",
    "og_downsample", "og_downsampled_desc", "og_downsampled_export", "og_downsampled_free",
    "og_downsample_shard", "og_downsampled_timing",
    "og_tssp_parse", "og_tssp_desc", "og_tssp_measurement", "og_tssp_time_range", "og_tssp_free",
    "og_shard_open_files", "og_shard_merge_info", "og_shard_append_files", "og_shard_compact",
    "og_shard_append_rows", "og_shard_open_rows",
    "og_shard_write_tssp", "og_tssp_image_size", "og_tssp_image_export", "og_tssp_image_timing", "og_tssp_image_free",
]

_lib = None


class OgpuError(RuntimeError):
    def __init__(self, status, where):
        self.status = status
        msg = lib().og_last_error().decode(errors="replace")
        super().__init__(f"{where}: {lib().og_strerror(status).decode()} ({status}) {msg}")


def lib():
    """Load libogpu.so; raise (never fall back) when it is missing."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(f"{LIB_PATH} is missing: run `python -c 'import __graft_entry__ as g; g.build()'` "
                           "(nvcc, sm_90a). There is no CPU fallback for the scan/aggregate path.")
    L = C.CDLL(LIB_PATH)
    L.og_strerror.restype = C.c_char_p
    L.og_strerror.argtypes = [C.c_int]
    L.og_last_error.restype = C.c_char_p
    L.og_version.restype = C.c_char_p
    L.og_init.argtypes = [C.c_int]
    L.og_shard_open.argtypes = [C.POINTER(ShardDesc), C.POINTER(C.c_void_p)]
    L.og_shard_open_files.argtypes = [C.POINTER(ShardDesc), u32p, C.c_uint32, C.POINTER(C.c_void_p)]
    L.og_shard_merge_info.argtypes = [C.c_void_p, C.POINTER(MergeInfo)]
    L.og_shard_append_files.argtypes = [C.c_void_p, C.POINTER(ShardDesc), u32p, C.c_uint32]
    L.og_shard_append_rows.argtypes = [C.c_void_p, C.POINTER(RowsDesc), C.POINTER(RowsInfo)]
    L.og_shard_open_rows.argtypes = [C.POINTER(RowsDesc), C.POINTER(C.c_void_p), C.POINTER(RowsInfo)]
    L.og_shard_compact.argtypes = [C.c_void_p, C.POINTER(CompactDesc), C.POINTER(CompactInfo)]
    L.og_shard_close.argtypes = [C.c_void_p]
    L.og_shard_close.restype = None
    L.og_shard_info.argtypes = [C.c_void_p, u64p, u64p, u64p, u64p, i64p, i64p]
    L.og_query_create.argtypes = [C.c_void_p, C.POINTER(QueryDesc), C.POINTER(C.c_void_p)]
    L.og_query_run.argtypes = [C.c_void_p]
    L.og_query_next.argtypes = [C.c_void_p, C.POINTER(RecordView)]
    L.og_query_dense.argtypes = [C.c_void_p, C.POINTER(DenseView)]
    L.og_query_stats.argtypes = [C.c_void_p, C.POINTER(Stats)]
    L.og_query_abort.argtypes = [C.c_void_p]
    L.og_query_abort.restype = None
    L.og_query_destroy.argtypes = [C.c_void_p]
    L.og_query_destroy.restype = None
    L.og_query_merge_dense.argtypes = [C.c_void_p, C.POINTER(DenseView)]
    L.og_decode_segment.argtypes = [C.c_void_p, C.c_uint32, C.POINTER(RecordView)]
    L.og_downsample.argtypes = [C.c_void_p, C.c_uint32, C.c_int64, C.c_int64, C.c_int64, C.POINTER(C.c_void_p)]
    L.og_downsample_shard.argtypes = [C.c_void_p, C.POINTER(DownsampleDesc), C.POINTER(C.c_void_p)]
    L.og_downsampled_timing.argtypes = [C.c_void_p, C.POINTER(C.c_double)]
    L.og_downsampled_desc.argtypes = [C.c_void_p, C.POINTER(ShardDesc), C.POINTER(C.c_uint64)]
    L.og_downsampled_export.argtypes = [C.c_void_p, C.c_void_p]
    L.og_downsampled_free.argtypes = [C.c_void_p]
    L.og_downsampled_free.restype = None
    L.og_tssp_parse.argtypes = [C.c_void_p, C.c_uint64, C.POINTER(C.c_void_p)]
    L.og_tssp_desc.argtypes = [C.c_void_p, C.POINTER(ShardDesc)]
    L.og_tssp_measurement.argtypes = [C.c_void_p]
    L.og_tssp_measurement.restype = C.c_char_p
    L.og_tssp_time_range.argtypes = [C.c_void_p, C.POINTER(C.c_int64), C.POINTER(C.c_int64)]
    L.og_tssp_free.argtypes = [C.c_void_p]
    L.og_tssp_free.restype = None
    L.og_shard_write_tssp.argtypes = [C.c_void_p, C.POINTER(TsspWriteDesc), C.POINTER(C.c_void_p)]
    L.og_tssp_image_size.argtypes = [C.c_void_p, u64p]
    L.og_tssp_image_export.argtypes = [C.c_void_p, C.c_void_p]
    L.og_tssp_image_timing.argtypes = [C.c_void_p, C.POINTER(C.c_double)]
    L.og_tssp_image_free.argtypes = [C.c_void_p]
    L.og_tssp_image_free.restype = None
    L.og_decode_segment_ex.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32, C.POINTER(RecordView)]
    L.og_decode_column_device.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint32, C.c_void_p, C.c_uint64, C.c_void_p]
    L.og_shard_synth.argtypes = [C.POINTER(SynthDesc), C.POINTER(C.c_void_p)]
    L.og_shard_layout_get.argtypes = [C.c_void_p, C.POINTER(ShardLayout)]
    L.og_shard_export.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    L.og_encode_pages.argtypes = [C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.c_uint32,
                                  C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p, u64p]
    L.og_comm_unique_id.argtypes = [C.c_void_p]
    L.og_comm_init_rank.argtypes = [C.c_void_p, C.c_int, C.c_int, C.POINTER(C.c_void_p)]
    L.og_comm_destroy.argtypes = [C.c_void_p]
    L.og_comm_destroy.restype = None
    L.og_comm_info.argtypes = [C.c_void_p, C.POINTER(C.c_int), C.POINTER(C.c_int), C.POINTER(C.c_int)]
    L.og_comm_allreduce_f64.argtypes = [C.c_void_p, C.POINTER(C.c_double), C.c_int, C.c_int]
    L.og_query_allreduce.argtypes = [C.c_void_p, C.c_void_p]
    _lib = L
    return L


def check(status, where):
    if status != OG_OK:
        raise OgpuError(status, where)
