/*
 * downsample.cu — the read-aggregate-write pass of a downsample / level compaction behind ONE C-ABI call (configs[4]).
 * Replaces engine/record_plan.go:494-830 (FileSequenceAggregator pulls records, newProcessor reduces them per series and window)
 * feeding engine/immutable/stream_downsample.go:454-600 (the downsampled columns go through the ordinary column builders,
 * column_builder.go:151-349, chunkdata_builder.go:65-97).
 *
 * Two entry points, one pass (downsample_pass):
 *   og_downsample_shard  every field column of the shard under a per-type call list, <call>_<field> columns sorted by name
 *   og_downsample        one numeric column with min, max, sum, count, first, last, columns <call>_f<column> in that order
 *
 * Everything heavy stays on the device; the host sees two numbers per series, a null flag per output column, and two i64 plus
 * one (offset, size) pair per output column per output segment.  The page bytes stay in HBM: og_downsampled_desc describes
 * them with OG_SHARD_DEVICE_DATA, so the new shard can be opened and queried in place, or copied out with og_downsampled_export
 * to be written to a file.
 */
#include <cub/block/block_reduce.cuh>
#include <cub/block/block_scan.cuh>
#include <cub/device/device_scan.cuh>

#include <algorithm>
#include <chrono>
#include <cstring>

#include <memory>
#include <string>
#include <vector>

#include "internal.h"

using namespace ogpu;

namespace {

constexpr uint32_t DS_ROWS = 1000; /* rows per segment of the output (lib/util/util.go:72) */
constexpr int DS_THREADS = 256;
const char *const FNAME[OG_AGG_LAST + 1] = {"", "count", "sum", "min", "max", "first", "last"};

struct DsxCol {            /* one output column */
    const uint64_t *src;   /* dense [series][window] 8-byte cells of the query that computed it */
    const uint8_t *src_ok; /* dense [series][window] validity */
    void *dst;             /* [n_seg * DS_ROWS] cells, segment-major: 8 B, or 1 B for bool (the forms og_encode_pages takes) */
    uint8_t *dst_ok;       /* [n_seg * DS_ROWS] one validity byte per row; og_encode_pages turns them into the page bitmap */
    int32_t bool_cells;
};

/* block per series: keep[s][b] = some output cell of series s in window b is non-null; rows_out[s] = kept windows,
 * segs_out[s] = the 1000-row segments they fill (segs_out[n_series] is left to the caller: 0, so the scan yields the total) */
__global__ void k_dsx_keep(const uint8_t *const *ok, uint32_t n_ok, uint32_t nb, uint8_t *keep, uint32_t *rows_out, uint64_t *segs_out) {
    typedef cub::BlockReduce<uint32_t, DS_THREADS> Reduce;
    __shared__ typename Reduce::TempStorage tmp;
    const size_t row0 = (size_t)blockIdx.x * nb;
    uint32_t n = 0;
    for (uint32_t b = threadIdx.x; b < nb; b += DS_THREADS) {
        uint8_t k = 0;
        for (uint32_t c = 0; c < n_ok; c++) k |= ok[c][row0 + b];
        keep[row0 + b] = k != 0;
        n += k != 0;
    }
    n = Reduce(tmp).Sum(n);
    if (threadIdx.x == 0) { rows_out[blockIdx.x] = n; segs_out[blockIdx.x] = (n + DS_ROWS - 1) / DS_ROWS; }
}

/* block per (series, output column); blockIdx.y == n_cols is the time column, which also writes each segment's row count and
 * time range.  Kept windows go, in time order, to rows [seg_base[s] * DS_ROWS + rank] of the column; col_nulls[c] is set when
 * column c has a null cell in a kept window. */
__global__ void k_dsx_scatter(const DsxCol *cols, uint32_t n_cols, const uint8_t *keep, uint32_t nb, int64_t start, int64_t interval,
                              const uint32_t *rows_s, const uint64_t *seg_base, int64_t *time, uint32_t *seg_rows, int64_t *seg_tmin,
                              int64_t *seg_tmax, uint32_t *col_nulls) {
    typedef cub::BlockScan<uint32_t, DS_THREADS> Scan;
    __shared__ typename Scan::TempStorage tmp;
    __shared__ uint32_t carry;
    const uint32_t s = blockIdx.x, n = rows_s[s];
    if (n == 0) return; /* block-uniform */
    const bool is_time = blockIdx.y == n_cols;
    const size_t row0 = (size_t)s * nb;
    const uint64_t seg0 = seg_base[s], base = seg0 * DS_ROWS;
    DsxCol col{};
    if (!is_time) col = cols[blockIdx.y];
    else for (uint32_t g = threadIdx.x; g * DS_ROWS < n; g += DS_THREADS) seg_rows[seg0 + g] = min(DS_ROWS, n - g * DS_ROWS);
    if (threadIdx.x == 0) carry = 0;
    __syncthreads();
    for (uint32_t b0 = 0; b0 < nb; b0 += DS_THREADS) {
        const uint32_t b = b0 + threadIdx.x;
        const uint32_t k = (b < nb && keep[row0 + b]) ? 1u : 0u;
        uint32_t rank, total;
        Scan(tmp).ExclusiveSum(k, rank, total);
        const uint32_t before = carry;
        if (k) {
            const uint32_t r = before + rank;
            const uint64_t at = base + r;
            if (is_time) {
                const int64_t t = start + (int64_t)b * interval;
                time[at] = t;
                if (r % DS_ROWS == 0) seg_tmin[seg0 + r / DS_ROWS] = t;
                if (r % DS_ROWS == DS_ROWS - 1 || r == n - 1) seg_tmax[seg0 + r / DS_ROWS] = t;
            } else {
                const uint8_t ok = col.src_ok[row0 + b];
                const uint64_t v = ok ? col.src[row0 + b] : 0;
                if (col.bool_cells) ((uint8_t *)col.dst)[at] = v != 0;
                else ((uint64_t *)col.dst)[at] = v;
                col.dst_ok[at] = ok;
                if (!ok) col_nulls[blockIdx.y] = 1;
            }
        }
        __syncthreads(); /* everyone has read carry and is done with tmp */
        if (threadIdx.x == 0) carry = before + total;
        __syncthreads();
        if (carry == n) break; /* block-uniform: the series' last kept window is placed */
    }
}

/* one output column: the cells of call `call` of query `query` (indices into downsample_pass's call lists) */
struct OutCol { std::string name; int32_t type; uint32_t query, call; };

} // namespace

struct og_downsampled {
    uint8_t *d_data = nullptr; uint64_t data_len = 0;
    uint64_t rows = 0;
    std::vector<uint64_t> sids; std::vector<uint32_t> ssb;
    std::vector<int64_t> tmin, tmax;
    std::vector<std::vector<uint64_t>> off; std::vector<std::vector<uint32_t>> len; /* [n_columns + 1], time last */
    std::vector<std::string> names; std::vector<int32_t> types;
    std::vector<og_column_desc> cols;
    double phase_ms[4] = {0, 0, 0, 0}; /* queries, keep + scatter, encode, directory assembly */
    ~og_downsampled() { dev_free(d_data); }
};

/* The pass behind both entry points: one og_query per list in `qcalls`, the output columns `oc` taken from their results.
 *   1. one og_query per call list (OG_GROUP_PER_SERIES, the same range and interval): dense records that stay on the device;
 *      all of them lie on one grid
 *   2. k_dsx_keep: a series keeps a window where any of its output cells is non-null (empty windows are dropped,
 *      TransIntervalRec2Rec, lib/record/record.go:1298-1365); a device scan turns the 1000-row segments each series fills into
 *      segment offsets.  k_dsx_scatter: every output column's kept cells, and the time column (the window start), segment-major
 *   3. og_encode_pages per output column (with validity: pages of columns that are null in a kept window carry a bitmap) and for
 *      the time column
 *   4. the directory on the host, from per-series row counts and per-segment time ranges, page offsets and lengths */
static int downsample_pass(og_shard *s, int64_t interval, int64_t tmin, int64_t tmax, const std::vector<std::vector<og_call>> &qcalls,
                           const std::vector<OutCol> &oc, og_downsampled **out) {
    using clock = std::chrono::steady_clock;
    CU(cudaSetDevice(s->device));
    const auto t_start = clock::now();
    const uint32_t n_oc = (uint32_t)oc.size(), ns = s->n_series;

    std::unique_ptr<og_downsampled> r(new og_downsampled);
    r->sids = s->sids;
    r->ssb.assign((size_t)ns + 1, 0);
    r->off.resize(n_oc + 1); r->len.resize(n_oc + 1);
    for (const OutCol &c : oc) { r->names.push_back(c.name); r->types.push_back(c.type); }

    /* 1. one per-series query per call list, all created before any runs (so a refused range costs no device work) */
    std::vector<std::unique_ptr<og_query>> qs;
    std::vector<og_dense_view> dv(qcalls.size());
    for (const auto &calls : qcalls) {
        og_query_desc qd{};
        qd.interval = interval; qd.tmin = tmin; qd.tmax = tmax; qd.ascending = 1;
        qd.n_calls = (uint32_t)calls.size(); qd.calls = calls.data(); qd.group_mode = OG_GROUP_PER_SERIES;
        og_query *q = nullptr;
        int rc = og_query_create(s, &qd, &q);
        if (rc) return rc;
        qs.emplace_back(q);
    }
    for (size_t i = 0; i < qs.size(); i++) {
        int rc = og_query_run(qs[i].get());
        if (!rc) rc = og_query_dense(qs[i].get(), &dv[i]);
        if (rc) return rc;
        if (dv[i].start != dv[0].start || dv[i].n_buckets != dv[0].n_buckets || dv[i].interval != dv[0].interval || dv[i].n_groups != ns) {
            set_error("the queries of columns %u and 0 lie on different grids", (unsigned)i); return OG_E_STATE;
        }
    }
    r->phase_ms[0] = ms_since(t_start);
    const uint32_t nb = dv.empty() ? 0 : dv[0].n_buckets;
    Scratch tmp;
    uint32_t n_seg = 0;
    uint32_t *d_seg_rows = nullptr;
    int64_t *d_time = nullptr;
    std::vector<DsxCol> hcols(n_oc);
    std::vector<uint32_t> col_nulls(n_oc);
    if (n_oc && ns && nb) {
        /* 2. kept windows, segment offsets, scatter */
        auto t2 = clock::now();
        const uint8_t **d_okp = nullptr; uint8_t *d_keep = nullptr; uint32_t *d_rows = nullptr; uint64_t *d_segs = nullptr, *d_base = nullptr;
        std::vector<const uint8_t *> okp(n_oc);
        for (uint32_t c = 0; c < n_oc; c++) okp[c] = dv[oc[c].query].cols[oc[c].call].valid;
        int rc;
        if ((rc = tmp.get(&d_okp, n_oc)) || (rc = tmp.get(&d_keep, (size_t)ns * nb)) || (rc = tmp.get(&d_rows, ns)) ||
            (rc = tmp.get(&d_segs, (size_t)ns + 1)) || (rc = tmp.get(&d_base, (size_t)ns + 1))) return rc;
        CU(cudaMemcpy(d_okp, okp.data(), n_oc * sizeof(void *), cudaMemcpyHostToDevice));
        CU(cudaMemset(d_segs + ns, 0, 8));
        k_dsx_keep<<<ns, DS_THREADS>>>(d_okp, n_oc, nb, d_keep, d_rows, d_segs);
        CU(cudaGetLastError());
        size_t scan_bytes = 0; uint8_t *d_scan = nullptr;
        CU(cub::DeviceScan::ExclusiveSum(nullptr, scan_bytes, d_segs, d_base, ns + 1));
        if ((rc = tmp.get(&d_scan, scan_bytes))) return rc;
        CU(cub::DeviceScan::ExclusiveSum(d_scan, scan_bytes, d_segs, d_base, ns + 1));
        std::vector<uint32_t> rows_s(ns); std::vector<uint64_t> base(ns + 1);
        CU(cudaMemcpy(rows_s.data(), d_rows, (size_t)ns * 4, cudaMemcpyDeviceToHost));
        CU(cudaMemcpy(base.data(), d_base, ((size_t)ns + 1) * 8, cudaMemcpyDeviceToHost));
        if (base[ns] > 0xfffffff0ull) { set_error("too many output segments"); return OG_E_UNSUPPORTED; }
        n_seg = (uint32_t)base[ns];
        for (uint32_t i = 0; i < ns; i++) { r->ssb[i + 1] = (uint32_t)base[i + 1]; r->rows += rows_s[i]; }
        if (n_seg) {
            const uint64_t cells = (uint64_t)n_seg * DS_ROWS;
            int64_t *d_tmin = nullptr, *d_tmax = nullptr; DsxCol *d_cols = nullptr; uint32_t *d_nulls = nullptr;
            for (uint32_t c = 0; c < n_oc; c++) {
                const bool b1 = oc[c].type == OG_TYPE_BOOL;
                uint8_t *dst = nullptr, *dst_ok = nullptr;
                if ((rc = tmp.get(&dst, cells * (b1 ? 1 : 8))) || (rc = tmp.get(&dst_ok, cells))) return rc;
                /* cells past a series' last row are never encoded, but keep them defined */
                CU(cudaMemset(dst, 0, cells * (b1 ? 1 : 8))); CU(cudaMemset(dst_ok, 0, cells));
                const og_dense_col &dc = dv[oc[c].query].cols[oc[c].call];
                hcols[c] = DsxCol{(const uint64_t *)dc.values, dc.valid, dst, dst_ok, b1 ? 1 : 0};
            }
            if ((rc = tmp.get(&d_cols, n_oc)) || (rc = tmp.get(&d_time, cells)) || (rc = tmp.get(&d_seg_rows, n_seg)) ||
                (rc = tmp.get(&d_tmin, n_seg)) || (rc = tmp.get(&d_tmax, n_seg)) || (rc = tmp.get(&d_nulls, n_oc))) return rc;
            CU(cudaMemcpy(d_cols, hcols.data(), n_oc * sizeof(DsxCol), cudaMemcpyHostToDevice));
            CU(cudaMemset(d_time, 0, cells * 8));
            CU(cudaMemset(d_nulls, 0, n_oc * 4));
            k_dsx_scatter<<<dim3(ns, n_oc + 1), DS_THREADS>>>(d_cols, n_oc, d_keep, nb, dv[0].start, dv[0].interval, d_rows, d_base, d_time,
                                                              d_seg_rows, d_tmin, d_tmax, d_nulls);
            CU(cudaGetLastError());
            r->tmin.resize(n_seg); r->tmax.resize(n_seg);
            CU(cudaMemcpy(r->tmin.data(), d_tmin, (size_t)n_seg * 8, cudaMemcpyDeviceToHost));
            CU(cudaMemcpy(r->tmax.data(), d_tmax, (size_t)n_seg * 8, cudaMemcpyDeviceToHost));
            CU(cudaMemcpy(col_nulls.data(), d_nulls, n_oc * 4, cudaMemcpyDeviceToHost));
        }
        qs.clear(); /* the dense records have been read */
        r->phase_ms[1] = ms_since(t2);
    }
    auto t4 = clock::now();
    if (n_seg) {
        /* 3. encode every output column, then time, into one scratch region.  A column without null cells goes without its
         *    validity bytes: the pages are the same, and the encoder skips a read per row (and, for int, a compacting copy). */
        auto t3 = clock::now();
        const uint64_t cap_col = (uint64_t)n_seg * 8800; /* a 1000-row page never exceeds 8 B per row + headers */
        const uint64_t bound = cap_col * (n_oc + 1);
        uint8_t *d_pages = nullptr; uint64_t *d_off = nullptr; uint32_t *d_len = nullptr;
        int rc;
        if ((rc = tmp.get(&d_pages, bound)) || (rc = tmp.get(&d_off, (size_t)(n_oc + 1) * n_seg)) || (rc = tmp.get(&d_len, (size_t)(n_oc + 1) * n_seg))) return rc;
        std::vector<uint64_t> col_pos(n_oc + 1);
        uint64_t pos = 0;
        for (uint32_t c = 0; c <= n_oc; c++) {
            const bool is_time = c == n_oc;
            uint64_t bytes = 0;
            col_pos[c] = pos;
            rc = og_encode_pages(is_time ? OG_TYPE_INT : oc[c].type, is_time ? 1 : 0, is_time ? (const void *)d_time : hcols[c].dst,
                                 is_time || !col_nulls[c] ? nullptr : hcols[c].dst_ok, d_seg_rows, n_seg, DS_ROWS, d_pages + pos, bound - pos,
                                 d_off + (size_t)c * n_seg, d_len + (size_t)c * n_seg, &bytes);
            if (rc) return rc;
            pos += bytes;
        }
        r->phase_ms[2] = ms_since(t3);
        /* 4. directory + one exact-size data region (with the slack word-granular readers need behind the last page) */
        t4 = clock::now();
        std::vector<uint64_t> off((size_t)(n_oc + 1) * n_seg); std::vector<uint32_t> len(off.size());
        CU(cudaMemcpy(off.data(), d_off, off.size() * 8, cudaMemcpyDeviceToHost));
        CU(cudaMemcpy(len.data(), d_len, len.size() * 4, cudaMemcpyDeviceToHost));
        for (uint32_t c = 0; c <= n_oc; c++) {
            r->off[c].assign(off.begin() + (size_t)c * n_seg, off.begin() + (size_t)(c + 1) * n_seg);
            r->len[c].assign(len.begin() + (size_t)c * n_seg, len.begin() + (size_t)(c + 1) * n_seg);
            for (uint64_t &o : r->off[c]) o += col_pos[c];
        }
        if ((rc = dalloc(&r->d_data, pos + 1024))) return rc;
        r->data_len = pos;
        CU(cudaMemcpy(r->d_data, d_pages, pos, cudaMemcpyDeviceToDevice));
        CU(cudaMemset(r->d_data + pos, 0, 1024));
    }
    if (!r->d_data) { /* nothing survived: an empty shard still has a valid (zero-length) data region */
        if (int rc = dalloc(&r->d_data, 1024)) return rc;
        r->data_len = 0;
        CU(cudaMemset(r->d_data, 0, 1024));
    }
    for (uint32_t c = 0; c < n_oc; c++) {
        og_column_desc cd; cd.name = r->names[c].c_str(); cd.type = r->types[c]; cd.page_off = r->off[c].data(); cd.page_len = r->len[c].data();
        r->cols.push_back(cd);
    }
    CU(cudaDeviceSynchronize());
    r->phase_ms[3] = ms_since(t4);
    *out = r.release();
    return OG_OK;
}

extern "C" {

OG_API void og_downsampled_free(og_downsampled *d) { delete d; }

OG_API int og_downsample(og_shard *s, uint32_t column, int64_t interval, int64_t tmin, int64_t tmax, og_downsampled **out) {
    if (!s || !out || interval <= 0) { set_error("bad argument (interval must be > 0)"); return OG_E_INVAL; }
    *out = nullptr;
    if (column >= s->n_columns) { set_error("column %u out of range", column); return OG_E_INVAL; }
    const int32_t ctype = s->col_types[column];
    if (ctype != OG_TYPE_FLOAT && ctype != OG_TYPE_INT) { set_error("downsample of a column of type %d", ctype); return OG_E_UNSUPPORTED; }
    static const int32_t funcs[] = {OG_AGG_MIN, OG_AGG_MAX, OG_AGG_SUM, OG_AGG_COUNT, OG_AGG_FIRST, OG_AGG_LAST};
    std::vector<std::vector<og_call>> qcalls(1);
    std::vector<OutCol> oc;
    for (uint32_t k = 0; k < 6; k++) {
        qcalls[0].push_back({funcs[k], (int32_t)column});
        oc.push_back({std::string(FNAME[funcs[k]]) + "_f" + std::to_string(column), funcs[k] == OG_AGG_COUNT ? OG_TYPE_INT : ctype, 0, k});
    }
    return downsample_pass(s, interval, tmin, tmax, qcalls, oc, out);
}

/* og_downsample_shard: every field column of the shard under the policy's per-type call lists, in one pass */
OG_API int og_downsample_shard(og_shard *s, const og_downsample_desc *d, og_downsampled **out) {
    if (!s || !d || !out) { set_error("null argument"); return OG_E_INVAL; }
    *out = nullptr;
    if (d->interval <= 0 || d->tmin > d->tmax) { set_error("bad argument (interval must be > 0 and tmin <= tmax)"); return OG_E_INVAL; }
    if (d->n_types && !d->ops) { set_error("n_types is %u but ops is NULL", d->n_types); return OG_E_INVAL; }

    /* the policy: at most one call list per type, each call at most once, and only calls the type has a reducer for */
    const og_downsample_ops *by_type[OG_TYPE_BOOL + 1] = {};
    for (uint32_t i = 0; i < d->n_types; i++) {
        const og_downsample_ops &o = d->ops[i];
        if (o.type != OG_TYPE_INT && o.type != OG_TYPE_FLOAT && o.type != OG_TYPE_STRING && o.type != OG_TYPE_BOOL) { set_error("ops[%u]: unknown field type %d", i, o.type); return OG_E_INVAL; }
        if (by_type[o.type]) { set_error("ops[%u]: a second call list for field type %d", i, o.type); return OG_E_INVAL; }
        if (o.n_funcs && !o.funcs) { set_error("ops[%u]: n_funcs is %u but funcs is NULL", i, o.n_funcs); return OG_E_INVAL; }
        uint32_t seen = 0;
        for (uint32_t k = 0; k < o.n_funcs; k++) {
            const int32_t f = o.funcs[k];
            if (f < OG_AGG_COUNT || f > OG_AGG_LAST) { set_error("ops[%u].funcs[%u]: bad function %d", i, k, f); return OG_E_INVAL; }
            if (seen & (1u << f)) { set_error("ops[%u]: %s() listed twice", i, FNAME[f]); return OG_E_INVAL; }
            seen |= 1u << f;
            if (o.type == OG_TYPE_BOOL && f == OG_AGG_SUM) { set_error("ops[%u]: sum() over boolean fields (the reference has no boolean sum reducer)", i); return OG_E_INVAL; }
            if (o.type == OG_TYPE_STRING && f != OG_AGG_COUNT) {
                set_error("ops[%u]: %s() over string fields is not supported: only count() is, because string values are never decoded on the device", i, FNAME[f]);
                return OG_E_UNSUPPORTED;
            }
        }
        by_type[o.type] = &o;
    }

    /* output columns: <call>_<field> for every field whose type has calls, sorted by name (og_shard_desc's schema order) */
    std::vector<OutCol> oc;
    std::vector<std::vector<og_call>> qcalls; /* per source column, in the order of its type's call list */
    for (uint32_t c = 0; c < s->n_columns; c++) {
        const int32_t typ = s->col_types[c];
        const og_downsample_ops *o = typ >= 0 && typ <= OG_TYPE_BOOL ? by_type[typ] : nullptr;
        if (!o || o->n_funcs == 0) continue; /* a type without calls drops its fields */
        std::vector<og_call> calls;
        for (uint32_t k = 0; k < o->n_funcs; k++) {
            const int32_t f = o->funcs[k];
            oc.push_back({std::string(FNAME[f]) + "_" + s->col_names[c], f == OG_AGG_COUNT ? OG_TYPE_INT : typ, (uint32_t)qcalls.size(), k});
            calls.push_back({f, (int32_t)c});
        }
        qcalls.push_back(calls);
    }
    std::stable_sort(oc.begin(), oc.end(), [](const OutCol &a, const OutCol &b) { return a.name < b.name; });
    if (oc.size() + 1 > 65535) { set_error("%u output columns (at most 65534)", (unsigned)oc.size()); return OG_E_UNSUPPORTED; }
    return downsample_pass(s, d->interval, d->tmin, d->tmax, qcalls, oc, out);
}

OG_API int og_downsampled_timing(const og_downsampled *d, double phase_ms[4]) {
    if (!d || !phase_ms) { set_error("null argument"); return OG_E_INVAL; }
    for (int i = 0; i < 4; i++) phase_ms[i] = d->phase_ms[i];
    return OG_OK;
}

OG_API int og_downsampled_desc(const og_downsampled *d, og_shard_desc *desc, uint64_t *rows) {
    if (!d || !desc) { set_error("null argument"); return OG_E_INVAL; }
    memset(desc, 0, sizeof *desc);
    desc->data = d->d_data; desc->data_len = d->data_len;
    desc->n_series = (uint32_t)d->sids.size(); desc->sids = d->sids.data(); desc->series_seg_begin = d->ssb.data();
    desc->n_segments = (uint32_t)d->tmin.size(); desc->seg_tmin = d->tmin.data(); desc->seg_tmax = d->tmax.data();
    desc->n_columns = (uint32_t)d->cols.size(); desc->columns = d->cols.data();
    desc->time_page_off = d->off.back().data(); desc->time_page_len = d->len.back().data();
    desc->flags = OG_SHARD_DEVICE_DATA;
    if (rows) *rows = d->rows;
    return OG_OK;
}

OG_API int og_downsampled_export(const og_downsampled *d, uint8_t *host_data) {
    if (!d || !host_data) { set_error("null argument"); return OG_E_INVAL; }
    if (d->data_len == 0) return OG_OK;
    cudaError_t e = cudaMemcpy(host_data, d->d_data, d->data_len, cudaMemcpyDeviceToHost);
    return e == cudaSuccess ? OG_OK : cuda_fail(e, "og_downsampled_export", __FILE__, __LINE__);
}

} // extern "C"
