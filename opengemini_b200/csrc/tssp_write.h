/*
 * tssp_write.h — what the device half of the TSSP writer (tssp_write.cu) hands to the host half (tssp.cpp): per (series, column)
 * the pre-aggregation cell and the file offset of the column's CRC, per segment the page offsets and lengths.  Nothing per row.
 */
#pragma once
#include <cstdint>
#include <string>
#include <vector>

namespace ogpu {

/* pre-aggregation of one column of one chunk (engine/immutable/pre_aggregation.go): values as raw 64-bit cells (double bits,
 * int64, bool 0/1 with the builders' initial 2 / -1).  String and time columns use `count` only. */
struct PreAggCell { uint64_t minv, maxv; int64_t mint, maxt; uint64_t sum; int64_t count; };

struct TsspTailIn {
    const char *measurement;
    uint32_t n_series, n_segments, n_cols1;      /* series and segments of the written range; field columns + time */
    const uint64_t *sids;                        /* [n_series] */
    const uint32_t *seg_begin;                   /* [n_series + 1] first segment of each series, relative to the range */
    const int64_t *seg_tmin, *seg_tmax;          /* [n_segments] */
    const std::string *col_names;                /* [n_cols1 - 1] field columns in name order; time is last */
    const int32_t *col_types;                    /* [n_cols1 - 1] */
    const PreAggCell *cells;                     /* [n_series * n_cols1] */
    const uint8_t *col_present;                  /* [n_series * n_cols1] 1: the chunk holds the column */
    const uint64_t *chunk_off;                   /* [n_series + 1] file offset of each chunk; the last entry is the end of the data */
    const uint64_t *page_off;                    /* [n_cols1 * n_segments] file offset of each page */
    const uint32_t *page_len;                    /* [n_cols1 * n_segments] */
};

/* chunk-meta blocks, meta index, bloom filter, id-time section, trailer and footer of the file whose chunks end at
 * chunk_off[n_series] (tssp.cpp).  Returns an OG_* status with the error text set. */
int tssp_build_tail(const TsspTailIn &in, std::vector<uint8_t> &out);

} // namespace ogpu
