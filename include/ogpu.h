/*
 * ogpu.h — C ABI of libogpu.so: the H100 (sm_90a) scan/aggregate path behind openGemini's
 * cursor seam.  Plain pointers and sizes only; no C++/torch types cross this boundary.
 *
 * What each entry point replaces in the reference (paths relative to the openGemini tree):
 *
 *   og_shard_open            engine/immutable/tssp_reader.go:118,586 (TSSPFile.ReadAt: locate pages through
 *                            ChunkMeta.colMeta[i].entries[seg]{offset,size}, tssp_file_meta.go:60-63,377-385)
 *                            + lib/fileops/readcache page access.  Here: one upload of the data region + the
 *                            flattened ChunkMeta ("segment directory") into HBM.
 *   og_shard_open_files      the per-query merge of a shard's ordered and out-of-order files (engine/iterators.go:246,295,
 *                            agg_tagset_cursor.go:294-346,411-535, iterators_helper.go:484 mergeData), done once at open.
 *   og_tssp_parse/_desc      the directory half of the file open: footer -> trailer -> meta index -> chunk-meta blocks ->
 *                            ChunkMeta (engine/immutable/trailer.go:71-88, tssp_file_meta.go:606-687,789-802,
 *                            tssp_file.go:606-658); yields the og_shard_desc og_shard_open takes.  Host only.
 *   og_query_create/run      engine/iterators.go:130 shard.CreateCursor -> createGroupCursors :551 ->
 *                            NewAggregateCursor aggregate_cursor.go:65 + NewAggTagSetCursor agg_tagset_cursor.go:583;
 *                            SinkPlan (aggregate_cursor.go:208) builds what og_query_desc carries.
 *   og_query_next            comm.KeyCursor.Next / NextAggData (engine/comm/cursor.go:46-56) as drained by
 *                            ChunkReader.nextRecord (engine/iterator_plan.go:707-717): returns ColVal-shaped
 *                            views (lib/record/column.go:30-37) valid until the next call, like
 *                            record.CircularRecordPool (lib/record/record_pool.go:208-268).
 *   og_query_dense           the dense interval record AggTagSetCursor builds (agg_tagset_cursor.go:1012-1027,
 *                            lib/record/record.go:1327 BuildEmptyIntervalRec) — exposed as device arrays so the
 *                            cross-shard merge (engine/executor/rpc_transform.go:40-282 + agg_transform.go:248-304
 *                            in the reference) can be an NCCL all-reduce.
 *   og_decode_segment        engine/immutable/reader.go:674 decodeColumnData + append{Integer,Float,Boolean}Column
 *                            :504-579 + appendTimeColumnData :638 (Record materialisation for
 *                            HybridStoreReader-style callers, engine/hybrid_store_reader.go:444).
 *   og_encode_pages          engine/immutable/column_builder.go:151-349 enc*Column + EncodeColumnHeader :428,
 *                            chunkdata_builder.go:65 EncodeTime (downsample / compaction re-encode).
 *   og_downsample            engine/record_plan.go:494-830 + engine/immutable/stream_downsample.go:454-600: one column of a shard
 *                            -> per-series window aggregates -> re-encoded pages and their directory, in one call.
 *   og_downsample_shard      the same for every field of a shard under a per-type call list (services/downsample/functions.go:42-111,
 *                            executor/schema.go:1448-1475, engine/record_plan.go:256-420,494-830): <call>_<field> columns,
 *                            null cells where a field had no value in a kept window.
 *   og_shard_write_tssp      engine/immutable/msbuilder.go:1248-1303,1355-1433 (MsBuilder.WriteData / Flush), chunkdata_builder_ts.go:37-82
 *                            (EncodeChunk: per column [crc32][pages]), pre_aggregation.go (the pre-agg blob of every ColumnMeta): an
 *                            open shard -> the bytes of one TSSP file, chunks laid out and checksummed on the device.
 *   og_shard_synth           test/bench tooling: builds a synthetic shard directly in HBM with the encode kernels
 *                            (same bytes the oracle's restated encoders produce; see tests/test_gpu_parity.py::test_synth_pages_byte_exact).
 *
 * Conventions (modelled on the in-tree cgo precedents engine/index/textindex/textbuilder_c.h:20-28 and
 * lib/util/lifted/encoding/lz4/lz4_linux_amd64.go:18-30): opaque handles, caller-owned inputs, library-owned
 * outputs, int status returns, no callbacks, no retained caller pointers after a call returns (og_shard_open
 * copies what it needs).  A handle is confined to one thread at a time; distinct queries may run concurrently.
 * There is NO CPU fallback: every compute entry point returns OG_E_CUDA when no device is bound.
 */
#ifndef OGPU_H
#define OGPU_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define OG_API __attribute__((visibility("default")))

/* ---- status codes (errors are codes, never panics across cgo; SURVEY §5.3) ---- */
enum {
    OG_OK = 0,
    OG_EOF = 1,            /* og_query_next: end of stream, the (nil,nil,nil) of KeyCursor.Next */
    OG_E_INVAL = -1,       /* bad argument / descriptor */
    OG_E_CUDA = -2,        /* CUDA runtime failure or no device bound */
    OG_E_NOMEM = -3,
    OG_E_UNSUPPORTED = -4, /* codec tag / option recognised but not implemented on the GPU path (zstd, mlf, lz4, DST location) */
    OG_E_CORRUPT = -5,     /* page failed validation (lib/errno InvalidFloatBuffer etc.) */
    OG_E_ABORTED = -6,     /* og_query_abort was called (closedSignal, engine/immutable/read_context.go:68-70) */
    OG_E_TYPE = -7,        /* "type(%v) in table not eq select type(%v)" column_builder.go:466 */
    OG_E_STATE = -8        /* call sequence error (next before run, ...) */
};

/* ---- column types: influx.Field_Type_* (lib/util/lifted/vm/protoparser/influx/parser.go:1363-1370) ---- */
enum { OG_TYPE_INT = 1, OG_TYPE_FLOAT = 3, OG_TYPE_STRING = 4, OG_TYPE_BOOL = 5 };

/* ---- aggregate calls pushed down to the store (engine/series_call_processor.go:56-80).
 *      mean() never arrives: the planner rewrites it to sum/count (engine/executor/schema.go:376-418). ---- */
enum { OG_AGG_COUNT = 1, OG_AGG_SUM = 2, OG_AGG_MIN = 3, OG_AGG_MAX = 4, OG_AGG_FIRST = 5, OG_AGG_LAST = 6 };

/* ---- WHERE filter: RPN over per-column compare terms (lib/binaryfilterfunc/functions.go:632, lib/rpn) ---- */
enum { OG_F_TERM = 0, OG_F_AND = 1, OG_F_OR = 2 };
enum { OG_OP_LT = 0, OG_OP_LTE = 1, OG_OP_GT = 2, OG_OP_GTE = 3, OG_OP_EQ = 4, OG_OP_NEQ = 5 };

typedef struct og_filter_item {
    int32_t kind;           /* OG_F_TERM / OG_F_AND / OG_F_OR */
    int32_t column;         /* field column index (TERM only) */
    int32_t op;             /* OG_OP_* (TERM only) */
    int32_t const_is_float; /* 1: compare against fval (int columns are converted with Int64ToFloat64Slice, functions.go:439); 0: ival */
    double fval;
    int64_t ival;           /* int constant, or 0/1 for bool columns */
} og_filter_item;

typedef struct og_call {
    int32_t func;   /* OG_AGG_* */
    int32_t column; /* field column index in the shard */
} og_call;

enum { OG_GROUP_ALL = 0, OG_GROUP_PER_SERIES = 1, OG_GROUP_MAP = 2 };
enum {
    OG_Q_STRICT_ORDER = 1u << 0 /* cross-series float sums in strict series order: bit-exact with the reference's sequential
                                   merge (lib/record/reccord_functions.go:730-733).  Without it a one-tagset query on a regular
                                   shard folds the series of a lane group with warp shuffles first (a fixed, reproducible
                                   association; float sums then agree with the reference to ~1e-15 relative, inside the 1e-9
                                   bound; counts, min/max/first/last and their times stay bit-exact).  Tag groups and
                                   per-series output always use the strict order. */
    ,
    OG_Q_NO_FUSED = 1u << 1 /* force the generic materialise-tile path even when the fused kernel is eligible (testing / A-B) */
    ,
    OG_Q_NO_FAST = 1u << 2 /* fused path, but without the specialised Gorilla/const-delta kernel (testing / A-B) */
    ,
    OG_Q_RESERVED_8 = 1u << 3 /* was an A/B switch of the round-1 staging experiments; ignored */
    ,
    OG_Q_QUERY_GRID = 1u << 4 /* lay the dense interval record over the QUERY range [tmin, tmax] instead of its intersection with the
                                 shard's own time range (FileInfo.MinTime/MaxTime).  Every shard of a cross-shard query then builds the
                                 same (start, interval, n_buckets) grid, which og_query_merge_dense / og_query_allreduce require; the
                                 range must be bounded (not MinTime/MaxTime) */
};

typedef struct og_query_desc {
    int64_t interval;  /* GROUP BY time() duration in ns; 0 = no interval (one window = [tmin, tmax]) */
    int64_t offset;    /* hybridqp.Interval.Offset */
    int64_t tmin, tmax;/* inclusive query time range (util.TimeRange) */
    int32_t ascending; /* 1: ORDER BY time ASC; 0: ORDER BY time DESC (same windows and aggregates, og_query_next emits the latest
                          window first).  NOTE: a zero-initialised descriptor therefore asks for descending output. */
    uint32_t n_calls;
    const og_call *calls;
    uint32_t n_filter; /* 0 = no WHERE on fields */
    const og_filter_item *filter;
    int32_t group_mode; /* OG_GROUP_* : how series map to tagsets */
    uint32_t n_groups;  /* OG_GROUP_MAP only */
    const uint32_t *series_group; /* OG_GROUP_MAP: [n_series] group id per series (series order inside a group = shard order) */
    int32_t chunk_size; /* ChunkSizeNum: max rows per record returned by og_query_next (<=0: 1024) */
    uint32_t flags;     /* OG_Q_* */
} og_query_desc;

/* ---- shard description = TSSP data region + flattened ChunkMeta ---- */
typedef struct og_column_desc {
    const char *name;         /* column name (schema order = sorted by name, time last: lib/record/record.go:115-123) */
    int32_t type;             /* OG_TYPE_* */
    const uint64_t *page_off; /* [n_segments] byte offset of this column's page (segment) inside data; Segment.offset */
    const uint32_t *page_len; /* [n_segments] Segment.size; 0 = column absent in that chunk (all rows null) */
} og_column_desc;

enum {
    OG_SHARD_DEVICE_DATA = 1u << 0 /* `data` is a device pointer owned by the caller for the shard's lifetime (zero-copy);
                                      the allocation must extend >= 1024 readable bytes past data_len (word-granular over-reads of the last page) */
};

typedef struct og_shard_desc {
    const uint8_t *data; /* file bytes that the page offsets index (whole file or data region) */
    uint64_t data_len;
    uint32_t n_series;   /* chunks; one series id each (ChunkMeta.sid) */
    const uint64_t *sids;              /* [n_series] */
    const uint32_t *series_seg_begin;  /* [n_series+1] first segment index of each series; segments of a series are
                                          consecutive and time-ordered (chunkdata_builder_ts.go:36-82) */
    uint32_t n_segments;
    const int64_t *seg_tmin;           /* [n_segments] ChunkMeta.timeRange[seg] */
    const int64_t *seg_tmax;
    uint32_t n_columns;                /* field columns (time excluded) */
    const og_column_desc *columns;
    const uint64_t *time_page_off;     /* [n_segments] time column pages */
    const uint32_t *time_page_len;
    uint32_t flags;                    /* OG_SHARD_* */
} og_shard_desc;

/* ---- ColVal / Record views (lib/record/column.go:30-37, record.go:57-61) ---- */
typedef struct og_colval_view {
    const uint8_t *val;     /* non-null values only, densely packed LE — both for decoded segments (reader.go:504-579) and for the
                               records og_query_next slices out of the interval record (TransIntervalRec2Rec, record.go:1340-1358) */
    uint64_t val_bytes;
    const uint8_t *bitmap;  /* LSB-first, 1 = present, bit index = bitmap_offset + row (column.go:26-28,489-498) */
    const int64_t *times;   /* RecMeta.Times[col] for first/last in multi-call queries, else NULL */
    int32_t type;           /* OG_TYPE_* of the output column (count -> INT) */
    int32_t len;
    int32_t nil_count;
    int32_t bitmap_offset;
} og_colval_view;

typedef struct og_record_view {
    uint32_t n_cols;
    const og_colval_view *cols; /* field columns in call order */
    const int64_t *times;       /* time column (always full) */
    int32_t rows;
    uint32_t group;             /* tagset / group id this record belongs to */
    uint64_t sid;               /* OG_GROUP_PER_SERIES: series id */
} og_record_view;

/* dense interval record on the device: what leaves AggTagSetCursor before TransIntervalRec2Rec */
typedef struct og_dense_col {
    void *values;    /* device, [n_groups * n_buckets] 8-byte cells (bool min/max/first/last stored as int64 0/1) */
    uint8_t *valid;  /* device, [n_groups * n_buckets] 1 = non-null */
    int64_t *times;  /* device, [n_groups * n_buckets] row time carried by selectors (min/max/first/last); NULL for sum/count */
    int32_t type;    /* OG_TYPE_* of the value cells */
    int32_t func;
} og_dense_col;

typedef struct og_dense_view {
    uint32_t n_groups;
    uint32_t n_buckets;
    int64_t start;     /* window start of bucket 0 (TimeWindowsInit, agg_tagset_cursor.go:1012) */
    int64_t interval;
    uint32_t n_cols;
    const og_dense_col *cols; /* host array of device pointers */
    void *stream;      /* cudaStream_t the arrays were produced on (already synchronised when run returns) */
} og_dense_view;

typedef struct og_stats {
    uint64_t rows_decoded;     /* rows in every decoded segment (SURVEY §8d row definition) */
    uint64_t segments_scanned; /* after time-range pruning (location.go:276-280) */
    uint64_t page_bytes;       /* algorithmic input bytes: value + time pages of scanned segments */
    uint64_t dir_bytes;        /* directory bytes read */
    uint64_t out_bytes;        /* dense output bytes */
    double kernel_ms;          /* device time of the last og_query_run (CUDA events on the query stream) */
    double h2d_ms;
    double main_kernel_ms;     /* of which: the dominant decode+reduce kernel(s) (k_fused_segment, or decode/filter/reduce tiles) */
    uint32_t kernel_launches;  /* kernels launched by the last og_query_run */
    int32_t path;              /* 0 generic materialise-tile path; 4 fused multi-column / WHERE kernel (pull iterators, nothing
                                  materialised); 5 the column-at-a-time form of it (const-delta time pages, at most one WHERE
                                  term: k_fused_cols); 1 fused, general per-segment kernel only; 2 fused Gorilla kernel over the
                                  lane-interleaved copy with per-series cells (strict order / tag groups / per-series output);
                                  3 the same with interior windows folded in-warp (one tagset, regular shard) */
    int32_t il_state;          /* lane-interleaved copy of the queried float column: 1 ready, 0 not applicable, -1 no eligible page,
                                  -2 NOT BUILT for lack of device memory (the query ran on the slower general kernel) */
    int32_t per_series_cells_used; /* path 3 only: some lane group left the folded path (lanes out of step or irregular time grid) */
    double il_build_ms;        /* one-off cost of building that copy (first query on the column) */
    uint64_t il_bytes;         /* its size in HBM */
    uint64_t general_segments; /* segments of the column that the Gorilla kernel does not take (other codecs, nulls, irregular time pages) */
    double merge_ms;           /* device time of the last og_query_allreduce (pack + collectives + fold) */
    uint64_t il_packed_segments; /* segments of that copy stored as fixed-width XOR deltas rather than Gorilla records */
} og_stats;

typedef struct og_shard og_shard;
typedef struct og_query og_query;

/* ---- lifecycle ---- */
OG_API int og_init(int device_ordinal);            /* bind the calling process to a device; idempotent */
OG_API int og_device_count(void);
OG_API const char *og_strerror(int status);
OG_API const char *og_last_error(void);            /* thread-local detail message of the last failing call */
OG_API const char *og_version(void);
/* Device buffers of closed shards and destroyed queries stay in the device's memory pool for reuse (open/close loops do not pay
 * cudaMalloc/cudaFree); this hands the unused part back to the driver. */
OG_API int og_release_cached_memory(void);

/* ---- TSSP container -> shard description (host only; csrc/tssp.cpp).  Replaces the directory half of the reference's file
 * open: footer -> Trailer.Unmarshal (engine/immutable/trailer.go:71-88, table_stat.go:51-84,144-207) -> MetaIndex.unmarshal
 * (tssp_file_meta.go:789-802) -> chunk-meta blocks (tssp_file.go:606-658) -> ChunkMeta.unmarshal (tssp_file_meta.go:606-687,
 * 248-303).  `file` must stay valid (and unchanged) until og_tssp_free; the description og_tssp_desc fills borrows from the
 * handle and from `file` (page offsets are absolute file offsets, Segment.offset), and is what og_shard_open takes.  Series may
 * have different columns: the description holds the union, sorted by name, page_len 0 where a chunk lacks the column.
 * Compressed chunk metas (ChunkMetaCompressFlag != 0) and detached files are refused with OG_E_UNSUPPORTED. ---- */
typedef struct og_tssp og_tssp;
OG_API int og_tssp_parse(const uint8_t *file, uint64_t len, og_tssp **out);
OG_API int og_tssp_desc(const og_tssp *t, og_shard_desc *out);
OG_API const char *og_tssp_measurement(const og_tssp *t);                 /* TableStat.name */
OG_API int og_tssp_time_range(const og_tssp *t, int64_t *min_time, int64_t *max_time); /* TableStat.minTime / maxTime */
OG_API void og_tssp_free(og_tssp *t);

/* ---- shard ---- */
OG_API int og_shard_open(const og_shard_desc *desc, og_shard **out);
OG_API void og_shard_close(og_shard *s); /* queries of a closed shard may still be destroyed (og_query_destroy), not run */
/* page_bytes: the field and time pages as the files stored them (a Snappy page at its stored size, though it is held transcoded
 * to a raw page) while every transcoded page is still in the shard, that is until the first append that merges rows or the first
 * compaction that re-cuts a series; from then on, later appends included, the pages as the shard holds them. */
OG_API int og_shard_info(const og_shard *s, uint64_t *n_series, uint64_t *n_segments, uint64_t *n_rows,
                         uint64_t *page_bytes, int64_t *tmin, int64_t *tmax);

/* ---- a shard's ordered and out-of-order files as ONE og_shard (csrc/merge.cu).  Replaces the per-query file-set read of the
 * reference: ordered files visited one after another (engine/agg_tagset_cursor.go:294-346), out-of-order files merged newest
 * first (agg_tagset_cursor.go:411-535, MergeRecordLimitRows), the result merged into the ordered records (engine/file_cursor.go:
 * 292-348 -> iterators_helper.go:484 mergeData -> lib/record/record.go:843 MergeRecordByMaxTimeOfOldRec), over the files that
 * immTables.GetBothFilesRef hands a query (engine/iterators.go:246,295).  Here the merge runs once, on the device, when the shard
 * is opened, and every query / decode / downsample / export entry point serves the result.
 *   files[]      in file-sequence order, oldest first (ordered and out-of-order files interleaved as they come); each is what
 *                og_tssp_desc or a caller builds for og_shard_open, with host data (OG_SHARD_DEVICE_DATA is refused here).
 *   file_flags[] OG_FILE_OUT_OF_ORDER marks the out-of-order files; every out-of-order file is newer than every ordered one.
 * Row rule (record.go:468-505 mergeRecRow): where files hold the same series and time, each column takes the newest file's value,
 * the older one's when that is null.  The schema is the union of the field columns by name, sorted by name (record.go:438-466); a
 * column a file lacks is null for its rows.  Series are the union by sid, ascending.
 * Only the rows of a series around its out-of-order rows are re-encoded (1000-row segments, the encoders of og_encode_pages; a
 * float segment the Gorilla encoder refuses gets a raw page): ordered segments outside that span keep their bytes.  The shard's
 * data region holds the pages its directory references; without out-of-order rows it is the files' bytes as they were copied in.
 * Refused: a column with two types (OG_E_TYPE), ordered files that overlap in time for one series, a string column with values
 * inside a re-encoded span (OG_E_UNSUPPORTED), a time repeated within one file's series inside a span (OG_E_CORRUPT).
 * WHERE applies to the merged row (the reference filters each file before the merge: DESIGN.md "Deviations"). ---- */
enum { OG_FILE_OUT_OF_ORDER = 1u << 0 };
OG_API int og_shard_open_files(const og_shard_desc *files, const uint32_t *file_flags, uint32_t n_files, og_shard **out);
typedef struct og_merge_info {
    uint32_t n_files, n_out_of_order_files;
    uint64_t series_merged;          /* series that had out-of-order rows */
    uint64_t out_of_order_rows;      /* rows read from out-of-order files */
    uint64_t rows_replaced;          /* older rows whose time a newer file also holds */
    uint64_t rows_after_merge;
    uint64_t segments_kept;          /* ordered segments carried over byte for byte */
    uint64_t segments_rewritten_in, segments_rewritten_out;
    double merge_ms;                 /* elapsed time of the merge phase, from the splice of the spans' source segments to the gather
                                        of the live pages into the new data region (CUDA events on the legacy stream; includes the
                                        host work between batches) */
} og_merge_info;
OG_API int og_shard_merge_info(const og_shard *s, og_merge_info *out); /* og_shard_open / og_shard_synth shards: n_files = 1, zeros;
                                                                         after og_shard_append_files: that call's files and counters */

/* Adds files flushed after the shard was built.  files[] are in file-sequence order, oldest first, every one newer than every
 * file the shard holds; OG_FILE_OUT_OF_ORDER marks the out-of-order ones.  Afterwards the shard answers every entry point as
 * og_shard_open_files over its original files followed by these would, with one difference after out-of-order rows: each append
 * re-encodes the spans its own files touch, where the open re-encodes the hull of all of them, so the rewritten rows can be cut
 * into different segments.  og_shard_info's n_segments and page_bytes, the directory, and float sums of merged series (rounding)
 * may then differ from the open's; rows, counts, min / max / first / last and n_rows / tmin / tmax do not.
 *   The flush rule (engine/mutable/ts_table.go SplitRecordByTime): an appended ordered file's segments of a series start after
 *   the last time the shard holds for that series; one that does not is OG_E_UNSUPPORTED, naming the sid.
 *   Refused as og_shard_open_files refuses them, with the same statuses: a column with two types, OG_SHARD_DEVICE_DATA in files[],
 *   string values inside a re-encoded span, a time repeated within one file inside a span, corrupt pages.  While an og_query
 *   created on the shard is alive the call is OG_E_STATE (og_query_create on another thread waits while an append runs).
 *   On every error the shard stays as it was; only its interleaved copies may have been dropped (rebuilt on first use).
 *   Column and series indices move when a new name or sid sorts into the middle: rebuild series group maps after an append.
 *   Cost: the new files are copied in, validated and transcoded; spans are merged as at open; then the pages the new directory
 *   references are copied once, device to device, into a new data region (pages no longer referenced are left behind).  Peak
 *   device memory: about the live pages twice, plus the new files and the merge scratch.  A shard opened in place
 *   (OG_SHARD_DEVICE_DATA) gets its own buffer; the caller's buffer is never written. */
OG_API int og_shard_append_files(og_shard *s, const og_shard_desc *files, const uint32_t *file_flags, uint32_t n_files);

/* ---- rows into a shard: the flush of a memtable snapshot (csrc/flush.cu).  Replaces the device-side half of the reference's
 * memtable flush (engine/mutable/ts_table.go:63-133 FlushChunks): sort each series' record, split it at the series' last flushed
 * time, encode both parts into an ordered and an out-of-order file (MsBuilder.WriteRecord -> WriteData, engine/immutable/
 * msbuilder.go:1151), and add the files to the shard.  Here the rows go to the device once and are sorted, split and encoded
 * there; the files never exist on the host.
 *   Sort and deduplicate per series (WriteChunk.SortRecord -> ColumnSortHelper.Sort, lib/record/column_sort.go:42-97): rows
 *   sorted stably by time; for a run of equal times each column takes the last non-null value in arrival order, a null never
 *   replaces a value (replace, :100-107).
 *   Split (SplitRecordByTime, engine/mutable/ts_table.go:242-290): `last` is the latest time the shard holds for the series,
 *   INT64_MIN for a sid it lacks (MmsIdTime.get, engine/immutable/sequencer.go:92-101); rows with t > last form the ordered part,
 *   rows with t <= last the out-of-order part.  A column with no non-null value in a part is left out of that part (no page for
 *   the series in that file, ts_table.go:276-286), not written as an all-null page.
 *   Cut each part into 1000-row segments from its first row (WriteData; lib/util/util.go:72); every column kept in the part has
 *   a page in every segment, from the encoders of og_encode_pages (raw page for a float segment Gorilla refuses).
 *   Join the shard: afterwards the shard answers every entry point, byte for byte, as og_shard_append_files of those two files
 *   (ordered first, each only when it holds rows) would, og_shard_merge_info included (apart from merge_ms): the call reports
 *   as an append of its non-empty files.
 * Refused, the shard left as it was (only its interleaved copies may have been dropped; rebuilt on first use): a string field
 * (OG_E_UNSUPPORTED, naming it: there is no device string encoder); a field whose type differs from the shard's column of that
 * name (OG_E_TYPE); no rows, sid 0, a repeated sid or field name, a column whose len is neither 0 nor rows, a nil_count that
 * disagrees with the bitmap, val_bytes that disagree with len - nil_count, or non-zero flags (OG_E_INVAL); a live og_query of
 * the shard (OG_E_STATE; og_query_create on another thread waits while the flush runs).
 * Cost: one host-to-device copy per batch of series (batches under the merge's device-memory budget, each series charged its rows
 * and the 1000-row segment slots of its parts; OGPU_MERGE_BATCH_ROWS overrides the budget); the
 * out-of-order part is encoded here and decoded once more by the merge of og_shard_append_files. ---- */
typedef struct og_rows_field { const char *name; int32_t type; } og_rows_field; /* OG_TYPE_INT / FLOAT / BOOL */
typedef struct og_rows_series {
    uint64_t sid;               /* non-zero, unique in the call */
    uint32_t rows;
    const int64_t *times;       /* [rows] in arrival order: unsorted, equal times allowed */
    const og_colval_view *cols; /* [n_fields] in field order, the ColVal layout: val = non-null values packed densely (8 bytes
                                   each, 1 for bool), bitmap LSB-first from bitmap_offset (NULL allowed when nil_count == 0),
                                   len == rows, nil_count, type == the field's type, times NULL.  len == 0: the series has no
                                   such column in this call (all its rows null) */
} og_rows_series;
typedef struct og_rows_desc {
    uint32_t n_fields; const og_rows_field *fields; /* names unique */
    uint32_t n_series; const og_rows_series *series;
    uint32_t flags;                                 /* 0 */
} og_rows_desc;
typedef struct og_rows_info {
    uint64_t series_in, rows_in;
    uint64_t rows_replaced;     /* rows a later row of the same series and time replaced (deduplication inside the call) */
    uint64_t ordered_rows, out_of_order_rows;
    uint64_t segments_written;  /* segments of the two flushed files */
    double phase_ms[4];         /* wall clock: [0] rows staged and copied to the device, [1] expand + sort + split + runs of equal
                                   times, [2] combine + encode + the pages gathered into the two files, [3] add_files */
} og_rows_info;
OG_API int og_shard_append_rows(og_shard *s, const og_rows_desc *rows, og_rows_info *info /* may be NULL */);
/* a flush into an empty shard, as og_shard_open_files is an append to one */
OG_API int og_shard_open_rows(const og_rows_desc *rows, og_shard **out, og_rows_info *info /* may be NULL */);

/* ---- compaction of an open shard (csrc/compact.cu).  Replaces the device pass of the reference's non-streaming level
 * compaction (engine/immutable/compact.go:175-242): a series' merged records written through MsBuilder.WriteRecord -> WriteData
 * (msbuilder.go:1151), which cuts them into segments of R rows from the start of the series, every column of the chunk schema
 * (stream_compact.go:303 mergeSchema) with a page in every segment, null rows where a source lacked the column
 * (stream_compact.go:833-840 newNilCol).
 * A series is compact when every segment but its last holds R rows, its last 1..R, and every column has a page (an all-null page
 * counts) in every segment of the series or in none.  After the call every series is compact:
 *   a compact series keeps its directory entries and page bytes; a series with a column in only some segments is re-cut from
 *   its first segment; any other series is re-cut from its first segment that is not its last and holds fewer than R rows, or
 *   holds more than R rows (the segments before it end at multiples of R and keep their bytes).  Re-cut rows go into
 *   ceil(rows / R) new segments, every column of the series with a page in each (null where a source segment lacked it), pages
 *   from the encoders of og_encode_pages (raw page for a float segment Gorilla refuses), seg_tmin / seg_tmax from the rows.
 *   Rows, og_shard_info's n_rows / tmin / tmax and og_shard_merge_info are unchanged; n_segments and page_bytes are recomputed.
 *   An already compact shard is left untouched (no copy, every counter 0).
 * Refused, the shard left as it was (only its interleaved copies may have been dropped; rebuilt on first use):
 *   rows_per_segment above 1000 or non-zero flags (OG_E_INVAL); a string value inside a re-cut range (OG_E_UNSUPPORTED, naming
 *   the sid and the column: there is no device string encoder); a time that does not strictly ascend inside a re-cut range
 *   (OG_E_CORRUPT, naming the sid and the time); a live og_query of the shard (OG_E_STATE; og_query_create on another thread
 *   waits while a compaction runs).
 *   Cost: the re-cut rows are decoded into segment slots and encoded in batches under a device-memory budget, then the live pages
 *   are gathered into a new data region.  Peak device memory: about the live pages twice, plus one batch's scratch. */
typedef struct og_compact_desc {
    uint32_t rows_per_segment; /* R; 0 = 1000 (lib/util/util.go:72); 1..1000 (og_encode_pages' range); else OG_E_INVAL */
    uint32_t flags;            /* 0; anything else OG_E_INVAL */
} og_compact_desc;
typedef struct og_compact_info {
    uint64_t series_rewritten;                        /* series with at least one re-cut segment */
    uint64_t segments_kept;                           /* segments carried over byte for byte (0 when nothing was re-cut) */
    uint64_t segments_rewritten_in, segments_rewritten_out;
    uint64_t rows_rewritten;
    double compact_ms;                                /* CUDA events around the device pass, from the first decode to the gather
                                                         of the live pages (as og_merge_info.merge_ms) */
} og_compact_info;
OG_API int og_shard_compact(og_shard *s, const og_compact_desc *d, og_compact_info *info /* may be NULL */);

/* ---- query (aggregate cursor tree) ---- */
/* OG_E_UNSUPPORTED when the first or last row in range lies in a window that Window() clamps at the int64 time limits
 * (DESIGN.md "Deviations") */
OG_API int og_query_create(og_shard *s, const og_query_desc *desc, og_query **out);
OG_API int og_query_run(og_query *q);              /* launches the decode+aggregate kernels and waits for them */
OG_API int og_query_next(og_query *q, og_record_view *out); /* OG_OK + record, or OG_EOF */
OG_API int og_query_dense(og_query *q, og_dense_view *out);
OG_API int og_query_stats(const og_query *q, og_stats *out);
OG_API void og_query_abort(og_query *q);
OG_API void og_query_destroy(og_query *q);

/* merge another shard's dense partial (same query shape) into q's dense result on the device:
 * used after an all-gather for selector aggregates whose (value,time) tie-breaks are not a plain NCCL op
 * (lib/record/reccord_functions.go:482-494).  `other` holds device pointers laid out like og_query_dense's.
 * OG_E_INVAL, leaving q's record unchanged, when `other` differs in its shape, its grid (create both queries with
 * OG_Q_QUERY_GRID), which columns carry times, or in any column's func or type (as og_query_dense reports them: a count is
 * OG_TYPE_INT whatever column it counts, so counts of columns of different types merge). */
OG_API int og_query_merge_dense(og_query *q, const og_dense_view *other);

/* ---- cross-shard merge over NCCL (one shard per GPU, one process per GPU) ----
 * Replaces the exchange of per-shard partial aggregates between store and sql nodes (engine/executor/rpc_transform.go:40-282,
 * agg_transform.go:248-304).  Rank 0 makes an id with og_comm_unique_id and hands the 128 bytes to the other ranks through any
 * channel the host already has; every rank then calls og_comm_init_rank (collective).  og_query_allreduce (collective, same
 * query descriptor with OG_Q_QUERY_GRID on every rank) leaves the merged dense interval record on every rank: sums and counts
 * by ncclAllReduce, min/max/first/last by ncclAllGather + a fold in rank order with the reference's tie-breaks
 * (lib/record/reccord_functions.go:482-494).  NCCL is loaded with dlopen("libnccl.so.2") (override: OGPU_NCCL_LIB). */
typedef struct og_comm og_comm;
OG_API int og_comm_unique_id(uint8_t id[128]);
OG_API int og_comm_init_rank(const uint8_t id[128], int rank, int world, og_comm **out);
OG_API void og_comm_destroy(og_comm *c);
OG_API int og_comm_info(const og_comm *c, int *rank, int *world, int *nccl_version);
OG_API int og_comm_allreduce_f64(og_comm *c, double *vals, int n, int op_max); /* small host-side reduction (sum, or max when op_max) */
OG_API int og_query_allreduce(og_query *q, og_comm *c);

/* ---- materialise path (KeyCursor.Next for non-aggregating callers) ---- */
OG_API int og_decode_segment(og_shard *s, uint32_t segment, og_record_view *out);
/* flags: OG_DECODE_DESCENDING hands the segment over reversed — values, validity bits and times — as a descending scan does
 * (reader.go:516-519,1035-1042); callers walk the segments of a series from the last to the first (location.go:137-140,221-232) */
enum { OG_DECODE_DESCENDING = 1u << 0 };
OG_API int og_decode_segment_ex(og_shard *s, uint32_t segment, uint32_t flags, og_record_view *out);
/* decode a range of segments of one column into caller-provided DEVICE buffers (dense values, 8 B or 1 B each);
 * rows_out[i] receives the non-null value count of segment seg_begin+i. column == n_columns selects time. */
OG_API int og_decode_column_device(og_shard *s, uint32_t column, uint32_t seg_begin, uint32_t seg_end,
                                   void *d_values, uint64_t value_stride_bytes, uint32_t *d_rows_out);

/* ---- synthetic shard built on the device (bench/test tooling; uses the encode kernels) ---- */
enum { OG_SYNTH_F_HI = 0, OG_SYNTH_F_LO = 1, OG_SYNTH_INT_WALK = 2, OG_SYNTH_BOOL = 3 };
typedef struct og_synth_column {
    int32_t type;     /* OG_TYPE_* */
    int32_t dist;     /* OG_SYNTH_* */
    uint32_t null_permille; /* 0 = no nulls */
} og_synth_column;
typedef struct og_synth_desc {
    uint32_t n_series;
    uint32_t rows_per_series;
    uint32_t rows_per_segment; /* 1000 = lib/util/util.go:72 */
    int64_t t0;                /* first timestamp */
    int64_t dt;                /* cadence in ns (const-delta time pages) */
    uint64_t seed;
    uint32_t n_columns;
    const og_synth_column *columns;
    uint32_t series_base;      /* the shard holds series [series_base, series_base + n_series) of the synthetic population: the values
                                  of a series depend on (seed, column, series, row) only, so a small shard can reproduce any series
                                  of a large one (bench.py checks sampled series of the 10^10-row shard against the oracle this way) */
} og_synth_desc;
OG_API int og_shard_synth(const og_synth_desc *desc, og_shard **out);
/* copy a shard's pages + directory back to host (for parity tests against the oracle): caller passes buffers
 * sized from og_shard_info / og_shard_layout. */
typedef struct og_shard_layout {
    uint64_t data_len;
    uint32_t n_series, n_segments, n_columns;
} og_shard_layout;
OG_API int og_shard_layout_get(const og_shard *s, og_shard_layout *out);
OG_API int og_shard_export(const og_shard *s, uint8_t *data, uint64_t *sids, uint32_t *series_seg_begin,
                           int64_t *seg_tmin, int64_t *seg_tmax, uint64_t *page_off /*[(n_columns+1)*n_segments], time last*/,
                           uint32_t *page_len, int32_t *col_types /*[n_columns]*/);

/* ---- re-encode (downsample / compaction): encode dense device columns into pages ---- */
/* values: device [n_segments * rows_per_segment] 8-byte cells (bool: 1-byte cells), valid: device bitmap bytes per
 * segment or NULL (no nulls); out pages are written back to back into d_out (capacity out_cap) and their offsets /
 * lengths into d_page_off / d_page_len.  is_time selects EncodeTimestampBlock (chunkdata_builder.go:88-97). */
OG_API int og_encode_pages(int32_t type, int32_t is_time, const void *d_values, const uint8_t *d_valid,
                           const uint32_t *d_rows /*[n_segments] rows in each segment*/, uint32_t n_segments,
                           uint32_t rows_per_segment, uint8_t *d_out, uint64_t out_cap, uint64_t *d_page_off,
                           uint32_t *d_page_len, uint64_t *total_bytes_out);

/* ---- downsample / level compaction of one field column in one call (csrc/downsample.cu).  Replaces
 * engine/record_plan.go:494-830 (FileSequenceAggregator + newProcessor: per-series, per-window min/max/sum/count/first/last)
 * feeding engine/immutable/stream_downsample.go:454-600 (re-encode through the ordinary column builders).  The new shard has the
 * source's series, six field columns named min_f<c>, max_f<c>, sum_f<c>, count_f<c>, first_f<c>, last_f<c> (count is an integer
 * column, the others keep the source type), one row per window that held rows, the window start as row time, 1000-row
 * segments.  Its pages stay in device memory: og_downsampled_desc describes them with OG_SHARD_DEVICE_DATA (the description
 * borrows from the handle; open it with og_shard_open to query it in place), og_downsampled_export copies the page bytes to
 * the host for a file writer. ---- */
typedef struct og_downsampled og_downsampled;
OG_API int og_downsample(og_shard *s, uint32_t column, int64_t interval, int64_t tmin, int64_t tmax, og_downsampled **out);

/* ---- downsample a whole shard under a per-type policy (csrc/downsample.cu): what the reference's downsample task writes for one
 * shard of one measurement.  Replaces services/downsample/functions.go:42-111 (initDownSampleSchema: DownSamplePolicyInfo.GetCalls()
 * gives a call list per field type, applied to every field of that type; fields of a type without a list are dropped;
 * downSampleExprGen names each column <call>_<field>), executor/schema.go:1448-1475 (the output schema, addPrefix = true; count
 * is an integer column, the other calls keep the source type), engine/record_plan.go:256-420 (FieldIter / ChunkMetaByField read
 * a series one field at a time) and :494-830 (FileSequenceAggregator reduces per series and window, WriteIntoStorageTransform
 * writes the fields of a series against one time column).
 *   Calls by type: float, int: all six.  bool: count, min, max, first, last (sum is OG_E_INVAL: no boolean sum reducer).
 *   string: count only (any other call is OG_E_UNSUPPORTED: string values are never decoded on the device).  A type listed twice,
 *   a function outside OG_AGG_*, or a function listed twice in one list is OG_E_INVAL.  A type with an empty list is a type
 *   without a list.  A range whose first or last window is clamped at the int64 time limits is refused as og_query_create
 *   refuses it.
 *   Columns: one per (call, field) with calls, sorted by name; `og_shard_synth` shards name their fields f<c>.
 *   Rows: a series has one row per window in which ANY of its output cells is non-null, timed at the window start; a cell whose
 *   field had no non-null value in that window is null, and its page carries a bitmap.  (The reference gap-fills each field's
 *   windows with null rows across the series' time range, AppendRecWithNilRows record_plan.go:1234-1260, and so also writes rows
 *   that are null in every column; these are dropped here, as og_downsample drops empty windows.  DESIGN.md "Deviations".)
 *   Segments: 1000 rows; a series without rows in range has none.
 * The result is an ordinary og_downsampled handle: og_downsampled_desc / _export / _free serve it. ---- */
typedef struct og_downsample_ops {
    int32_t type;          /* OG_TYPE_* */
    uint32_t n_funcs;
    const int32_t *funcs;  /* [n_funcs] OG_AGG_* */
} og_downsample_ops;
typedef struct og_downsample_desc {
    int64_t interval, tmin, tmax;   /* window length (> 0) and inclusive time range, as og_downsample takes them */
    uint32_t n_types;
    const og_downsample_ops *ops;   /* [n_types] at most one entry per type; a type without an entry drops its fields */
} og_downsample_desc;
OG_API int og_downsample_shard(og_shard *s, const og_downsample_desc *d, og_downsampled **out);
/* wall-clock milliseconds of the phases of og_downsample and og_downsample_shard: [0] the per-column queries, [1] k_dsx_keep +
 * scan + k_dsx_scatter, [2] page encoding, [3] directory assembly and the output copy. */
OG_API int og_downsampled_timing(const og_downsampled *d, double phase_ms[4]);
OG_API int og_downsampled_desc(const og_downsampled *d, og_shard_desc *desc, uint64_t *rows /* may be NULL */);
OG_API int og_downsampled_export(const og_downsampled *d, uint8_t *host_data /* desc->data_len bytes */);
OG_API void og_downsampled_free(og_downsampled *d);

/* ---- an open shard as one TSSP file (csrc/tssp_write.cu, csrc/tssp.cpp).  Replaces, for data that is already on the device,
 * MsBuilder.WriteData / Flush (engine/immutable/msbuilder.go:1248-1303,1355-1433), TsChunkDataImp.EncodeChunk
 * (chunkdata_builder_ts.go:37-82), ChunkDataBuilder.EncodeTime (chunkdata_builder.go:65-114) and the pre-aggregation builders
 * (pre_aggregation.go).  Works on any og_shard: opened from a description or a file, synthesised, merged from a file set, or a
 * downsample result reopened in place (og_downsampled_desc -> og_shard_open).  The file is version 2, attached layout,
 * ChunkMetaCompressNone: header | chunks | chunk-meta blocks | meta index | bloom filter | id-time | trailer | footer, and
 * og_tssp_parse -> og_shard_open of its bytes gives back the shard's series, segments and pages.
 *   Pages are copied byte for byte; only pages the directory references are written (a merged shard's rewritten source pages
 *   stay behind; pages that were Snappy in the source were transcoded to raw pages at open, and those are written).  Every ColumnMeta carries the pre-aggregation blob of the column's rows as the reference's builders compute it
 *   (min / max with the time of their first occurrence, sum in row order, count; DESIGN.md lists what differs from the query
 *   reducers), every column of a chunk is prefixed by the CRC32 (IEEE) of its pages.
 *   A series without segments has no chunk.  A column whose page_len is 0 in every segment of a series is left out of that
 *   series' ChunkMeta, as the reference writes a series that lacks a field; all-null pages are pages and are listed.
 * Refused: an empty series range, a range none of whose series holds rows, series ids that are zero or not strictly ascending
 * (msbuilder.go:1252-1256) — OG_E_INVAL; a series with more than 65535 segments, a file above 8 GiB (engine/immutable/config.go:24-31,
 * lib/util/util.go:83), a column present in only some segments of a series, id-time values that the reference would encode
 * with zstd — OG_E_UNSUPPORTED, with text that says to narrow the series range where that helps; a page that does not decode —
 * OG_E_CORRUPT. ---- */
typedef struct og_tssp_write_desc {
    const char *measurement;            /* TableStat.name */
    uint32_t series_begin, series_end;  /* half-open range of the shard's series; 0,0 = all.  How a caller splits a shard that
                                           exceeds the per-file limits into several files */
    uint32_t flags;                     /* 0 */
} og_tssp_write_desc;
typedef struct og_tssp_image og_tssp_image;
OG_API int og_shard_write_tssp(og_shard *s, const og_tssp_write_desc *d, og_tssp_image **out);
OG_API int og_tssp_image_size(const og_tssp_image *f, uint64_t *bytes);
/* the whole file into `host` (og_tssp_image_size bytes): one device-to-host copy of the chunk region, the rest from host memory */
OG_API int og_tssp_image_export(const og_tssp_image *f, uint8_t *host);
/* wall-clock milliseconds of og_shard_write_tssp's phases: [0] pre-aggregation (k_preagg), [1] layout scan + k_tssp_gather +
 * k_tssp_crc_fold, [2] metadata to the host, [3] host assembly of everything behind the chunks */
OG_API int og_tssp_image_timing(const og_tssp_image *f, double phase_ms[4]);
OG_API void og_tssp_image_free(og_tssp_image *f);

#ifdef __cplusplus
}
#endif
#endif /* OGPU_H */
