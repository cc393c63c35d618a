/*
 * span_pass.h — what the two passes that re-encode rows of an open shard share: the merge of files into a shard (merge.cu) and
 * compaction (compact.cu).  Both decode spans of segments, write their rows into segment slots, encode them into a batch blob
 * under a device-memory budget, then splice the shard's kept segments and the new ones into one directory and gather the live
 * pages into a new data region.
 */
#pragma once
#include <cstdint>
#include <functional>
#include <string>
#include <vector>

#include "internal.h"

namespace ogpu {

#define MERGE_PAGE_BOUND 8704u /* largest page the encoders write for 1000 rows (encode.cu PAGE_STRIDE) */

/* the part of a device directory the decode kernels read */
struct SrcDir {
    const uint8_t *data; const uint64_t *page_off; const uint32_t *page_len; const uint32_t *seg_rows;
    uint32_t n_segments, n_columns;
};

enum { M_STRING = 100, M_REPEAT = 101 };
struct MergeErr { int code, seg, col, span, file; long long time; };

enum { SRC_SHARD = 0, SRC_FILES = 1, SRC_MERGED = 2 };
/* consecutive output segments [out0, next run's out0) of one series, from consecutive segments src0... of source `kind` */
struct Run { uint32_t out0, src0, series, kind; };

/* one source of spliced segments: a device directory whose column c is column col[c] of the source (-1: the source lacks it), or
 * column c itself when col is null */
struct SegSrc {
    const uint64_t *off; const uint32_t *len, *rows; const int64_t *tmin, *tmax;
    const uint32_t *seg_region; uint32_t region; /* data region of segment i: seg_region[i], or `region` when seg_region is null */
    const int32_t *col; uint32_t n_segments, n_columns;
};

struct NewSegs { /* what one batch produced, on the host */
    std::vector<uint64_t> off; std::vector<uint32_t> len; /* [(n_cols+1) * n] relative to the batch blob */
    std::vector<int64_t> tmin, tmax;
    std::vector<uint32_t> rows;
    uint8_t *blob = nullptr; uint64_t bytes = 0;
    uint32_t n = 0;
};

/* a spliced directory and the data region its pages were gathered into */
struct Spliced {
    uint32_t n = 0, n_columns = 0;
    uint64_t *off = nullptr; uint32_t *len = nullptr, *rows = nullptr, *series = nullptr; int64_t *tmin = nullptr, *tmax = nullptr;
    uint8_t *data = nullptr; uint64_t data_len = 0; /* null: the pages are in the files' region, at the offsets they have there */
};

/* *cap = rows one batch may hold: a quarter of the free device memory over `per_row` bytes, at least `floor_rows`; the
 * environment variable `env` (a test hook) replaces the budget */
int batch_cap_rows(uint64_t per_row, uint64_t floor_rows, const char *env, uint64_t *cap);

/* every non-string column of `types`, then the time column, of n segments (rows d_rows[g], row slots g * rps ...) encoded by the
 * og_encode_pages encoders (raw page for a float segment Gorilla refuses) into blob[*used, cap); ns.off / ns.len get each page's
 * place relative to the blob, *used grows by the bytes written */
int encode_columns(const std::vector<int32_t> &types, const int64_t *d_times, const std::vector<uint8_t *> &d_cols, const uint8_t *d_ok,
                   size_t out_rows, const uint32_t *d_rows, uint32_t n, uint32_t rps, uint8_t *blob, uint64_t cap, NewSegs &ns, uint64_t *used);
/* the end of a batch of ns.n new segments: their time ranges read back from d_tmin / d_tmax, their rows, and the first `used`
 * bytes of the batch's scratch blob kept in a buffer of `blobs` followed by 1024 zero bytes (k_append_gather reads past a page's
 * end), so the batch's scratch can go back to the pool before the next batch */
int keep_blob(const int64_t *d_tmin, const int64_t *d_tmax, std::vector<uint32_t> rows, const uint8_t *blob, uint64_t used, Scratch &blobs,
              NewSegs &ns);

#define MERGE_RPS 1000u /* rows per rewritten segment: lib/util/util.go:72 */

/* device scratch per row of a batch of nc columns: decode (8 t + 4 file + 4 span + 9 per column), sort (4 + 4 perm, 8 keys), heads +
   scan (8), output slots (8 + 9 per column), encoder staging and blob (2 x 8704 / 1000 per page) */
inline uint64_t span_row_bytes(uint32_t nc) { return 48 + 18ull * nc + 2ull * (nc + 1) * MERGE_PAGE_BOUND / MERGE_RPS + 64; }

/* The row rule over rows laid out span by span (span s at rows [span_row0[s], span_row0[s + 1]) of R), shared by the merge and the
 * flush (flush.cu):
 *   sort_spans          StableSortPairs by time inside each span: perm[i] = laid-out row of sorted row i (equal times keep their order)
 *   find_runs           k_merge_heads (row_file[perm[i]] repeated inside a run: M_REPEAT into *d_err), the exclusive scan of the
 *                       heads and each span's first output row (head, oidx, out_begin taken from `b`)
 *   combine_and_encode  k_merge_combine into 1000-row segment slots (each column takes its last non-null value in sorted order),
 *                       then encode_columns; ns gets the batch, seg_first[k] the first segment of span k in it ([n_spans + 1]).
 *                       span_has (may be null): [span][column] set where the column holds a value in the span. */
struct SortedRows {
    const int64_t *t; const uint32_t *perm, *row_span, *span_row0; /* row_span: by sorted position */
    const uint64_t *cells; const uint8_t *ok;                      /* [column][laid-out row] */
    uint32_t R, n_spans;
    uint32_t *head = nullptr, *oidx = nullptr, *out_begin = nullptr;
};
int sort_spans(const int64_t *times, int64_t *times_sorted, uint32_t *perm_in, uint32_t *perm, uint32_t R, uint32_t n_spans,
               const uint32_t *d_span_row0, Scratch &b);
int find_runs(SortedRows &r, const uint32_t *row_file, Scratch &b, MergeErr *d_err);
int combine_and_encode(const SortedRows &r, const std::vector<int32_t> &types, const int32_t *d_types, Scratch &b, unsigned long long *d_rep,
                       uint8_t *span_has, Scratch &blobs, NewSegs &ns, std::vector<uint32_t> &seg_first);

/* per series series[k] of `s`: last[k] its last time (INT64_MIN when it holds no segment) and, when `lo` / `hi` are given ([n]
 * each), [a[k], b[k]) the range of its segments that [lo[k], hi[k]] overlaps */
struct Probe { std::vector<int64_t> last; std::vector<uint32_t> a, b; };
int probe_series(const og_shard *s, const std::vector<uint32_t> &series, const int64_t *lo, const int64_t *hi, Probe &out);

/* pages from regions[page_region[p]] + src_off[p] to out + dst_off[p] (len[p] bytes each) with k_append_gather: the flush's
 * pages into the region of its files (flush.cu) */
int gather_pages(const std::vector<const uint8_t *> &regions, const std::vector<uint32_t> &page_region, const std::vector<uint64_t> &src_off,
                 const std::vector<uint32_t> &len, const std::vector<uint64_t> &dst_off, uint8_t *out);

/* New files whose pages are already on the device, as the flush (flush.cu) produces them: file f's pages at data + base[f], where
 * build_file_dir places a file set (16-byte aligned, back to back), followed by 1024 zero bytes; rows[] the rows of every segment,
 * files in order.  add_files takes the region over instead of copying host files in; the encoders wrote the pages, so they are
 * not validated again. */
struct DeviceFiles {
    uint8_t *data = nullptr; uint64_t data_len = 0;
    std::vector<uint32_t> rows;
    DeviceFiles() = default;
    DeviceFiles(const DeviceFiles &) = delete;
    DeviceFiles &operator=(const DeviceFiles &) = delete;
    ~DeviceFiles() { dev_free(data); }
};
/* files[] join `s` (og_shard_append_files; og_shard_open_files on an empty shard).  `who` names the caller in refusals.  dev: the
 * files' pages are on the device already (files[f].data is then never read) */
int add_files(og_shard *s, const og_shard_desc *files, const uint32_t *file_flags, uint32_t n_files, const char *who, DeviceFiles *dev);

/* The entry points that rewrite an open shard (og_shard_append_files, og_shard_append_rows, og_shard_compact): `pass` runs on the
 * shard's device under its live-query lock, so og_query_create waits until it is done; while a query lives the call is refused
 * with OG_E_STATE ("... destroy them before <verb>"). */
int rewrite_shard(og_shard *s, const char *verb, const std::function<int()> &pass);
/* The entry points that open a shard by a pass over an empty one (og_shard_open_files, og_shard_open_rows): the shard is created
 * on the library's device, `pass` runs on it, and it goes to *out when the pass succeeds */
int open_empty(og_shard **out, const std::function<int(og_shard *)> &pass);

/* the refusal of a string value inside a span `pass` re-encodes, or of a page that failed to decode in segment `seg` of `where` */
int string_refusal(unsigned long long sid, const std::string &column, const char *pass);
int decode_failure(int device_code, uint32_t seg, const char *where);

/* the new segments of every batch as one source directory (SRC_MERGED) over the pass's columns; batch b's blob is region
 * first_region + b, appended to `regions`.  m_first[b] is the first segment of batch b in it. */
int batches_source(const std::vector<NewSegs> &batches, uint32_t n_columns, uint32_t first_region, std::vector<const uint8_t *> &regions,
                   Scratch &own, SegSrc &out, std::vector<uint32_t> &m_first);

/* k_append_splice over `runs`, then the referenced pages gathered into one new buffer unless every run reads the files' region */
int splice_and_gather(const SegSrc src[3], const std::vector<Run> &runs, uint32_t n_out, uint32_t n_columns,
                      const std::vector<const uint8_t *> &regions, Scratch &own, Spliced &out);

/* n_rows, page_bytes, irregular_time_pages, max_seg_rows, tmin / tmax of a spliced directory (k_append_stats) into `out` */
int spliced_totals(const Spliced &sd, uint32_t n_columns, ShardState &out, const char *who);

/* The new state `out`, built apart, becomes s's.  The caller has run spliced_totals into `out` and set the fields its pass owns
 * (merge info, rows_merged, Snappy counters).  This completes the header from the series begin list, sids, column types and
 * names, uploads d_series_seg_begin and d_sids, hands sd's directory arrays and data region from `own` to `out`, synchronises,
 * swaps, and drops s's interleaved copies.  Nothing fails after the swap; on an earlier error `s` is as it was.  `out` leaves with
 * the old state, which it frees when the caller drops it (the caller's buffer of a shard opened in place is not freed). */
int install_state(og_shard *s, og_shard &out, Scratch &own, Spliced &sd, const std::vector<uint32_t> &series_seg_begin,
                  const std::vector<uint64_t> &sids, const std::vector<int32_t> &types, const std::vector<std::string> &names);

} // namespace ogpu
