/*
 * span_pass.h — what the two passes that re-encode rows of an open shard share: the merge of files into a shard (merge.cu) and
 * compaction (compact.cu).  Both decode spans of segments, write their rows into segment slots, encode them into a batch blob
 * under a device-memory budget, then splice the shard's kept segments and the new ones into one directory and gather the live
 * pages into a new data region.
 */
#pragma once
#include <cstdint>
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

/* one source of spliced segments: a device directory whose column c is column col[c] of the source (-1: the source lacks it) */
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
/* the first `used` bytes of a batch's scratch blob kept in a buffer of `blobs` followed by 1024 zero bytes (k_append_gather reads
 * past a page's end) */
int keep_blob(const uint8_t *blob, uint64_t used, Scratch &blobs, NewSegs &ns);

/* the refusal of a string value inside a span `pass` re-encodes, or of a page that failed to decode in segment `seg` of `where` */
int string_refusal(unsigned long long sid, const std::string &column, const char *pass);
int decode_failure(int device_code, uint32_t seg, const char *where);

/* the new segments of every batch as one source directory (SRC_MERGED); batch b's blob is region first_region + b, appended to
 * `regions`.  m_first[b] is the first segment of batch b in it. */
int batches_source(const std::vector<NewSegs> &batches, uint32_t n_columns, const int32_t *d_identity, uint32_t first_region,
                   std::vector<const uint8_t *> &regions, Scratch &own, SegSrc &out, std::vector<uint32_t> &m_first);

/* k_append_splice over `runs`, then the referenced pages gathered into one new buffer unless every run reads the files' region */
int splice_and_gather(const SegSrc src[3], const std::vector<Run> &runs, uint32_t n_out, uint32_t n_columns,
                      const std::vector<const uint8_t *> &regions, Scratch &own, Spliced &out);

/* n_rows, page_bytes, irregular_time_pages, max_seg_rows, tmin / tmax of a spliced directory (k_append_stats) into `out` */
int spliced_totals(const Spliced &sd, uint32_t n_columns, ShardState &out, const char *who);

/* the directory arrays and data region of `sd` handed from `own` to `out` */
void take_spliced(Scratch &own, Spliced &sd, ShardState &out);

} // namespace ogpu
