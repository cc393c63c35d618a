/*
 * api.cu — host side of libogpu.so: the C ABI declared in include/ogpu.h.
 * No CPU compute path exists here: every entry point that produces data launches kernels or fails with OG_E_CUDA.
 */
#include <algorithm>
#include <cstdarg>
#include <cstdio>
#include <cstring>
#include <numeric>

#include "agg_kernels.cuh"
#include "il_build.cuh"
#include "fused_multi.cuh"
#include "fused_cols.cuh"
#include "snappy_load.cuh"
#include <cub/device/device_scan.cuh>
#include <cub/device/device_radix_sort.cuh>
#include "internal.h"

namespace ogpu {

static thread_local char g_err[512] = "";
void set_error(const char *fmt, ...) {
    va_list ap; va_start(ap, fmt); vsnprintf(g_err, sizeof g_err, fmt, ap); va_end(ap);
}
int cuda_fail(cudaError_t e, const char *what, const char *file, int line) {
    set_error("CUDA error %d (%s) at %s:%d: %s", (int)e, cudaGetErrorString(e), file, line, what);
    return OG_E_CUDA;
}
static int g_device = -1;
cudaError_t dev_mem_info(size_t *free_b, size_t *total_b) {
    cudaError_t e = cudaMemGetInfo(free_b, total_b);
    if (e != cudaSuccess) return e;
    cudaMemPool_t pool; uint64_t reserved = 0, used = 0; int dev = 0;
    if (cudaGetDevice(&dev) == cudaSuccess && cudaDeviceGetDefaultMemPool(&pool, dev) == cudaSuccess &&
        cudaMemPoolGetAttribute(pool, cudaMemPoolAttrReservedMemCurrent, &reserved) == cudaSuccess &&
        cudaMemPoolGetAttribute(pool, cudaMemPoolAttrUsedMemCurrent, &used) == cudaSuccess && reserved > used) *free_b += (size_t)(reserved - used);
    else cudaGetLastError();
    return cudaSuccess;
}

int map_dev_err(int code) {
    switch (code) {
    case D_UNSUPPORTED: return OG_E_UNSUPPORTED;
    case D_TYPE: return OG_E_TYPE;
    case D_WATCHDOG: return OG_E_CUDA;
    default: return OG_E_CORRUPT;
    }
}

static DirP make_dir(const og_shard *s) {
    DirP d;
    d.data = s->d_data; d.page_off = s->d_page_off; d.page_len = s->d_page_len; d.seg_series = s->d_seg_series;
    d.seg_rows = s->d_seg_rows; d.series_seg_begin = s->d_series_seg_begin; d.seg_tmin = s->d_tmin; d.seg_tmax = s->d_tmax;
    d.n_segments = s->n_segments; d.n_columns = s->n_columns;
    return d;
}

/* derive seg_series / seg_rows / totals and validate codecs; shared by og_shard_open and og_shard_synth */
int shard_finalize(og_shard *s, bool scan_snappy) {
    int rc;
    s->il.resize(s->n_columns); /* sized once here: queries only read/lock individual entries later */
    if ((rc = dalloc(&s->d_seg_series, s->n_segments))) return rc;
    if ((rc = dalloc(&s->d_seg_rows, s->n_segments))) return rc;
    Scratch tmp;
    int32_t *d_types; unsigned long long *d_tot; uint32_t *d_max; int *d_err;
    if ((rc = tmp.get(&d_types, s->n_columns)) || (rc = tmp.get(&d_tot, 3)) || (rc = tmp.get(&d_max, 1)) || (rc = tmp.get(&d_err, 2))) return rc;
    CU(cudaMemcpy(d_types, s->col_types.data(), s->n_columns * sizeof(int32_t), cudaMemcpyHostToDevice));
    CU(cudaMemset(d_tot, 0, 24)); CU(cudaMemset(d_max, 0, 4)); CU(cudaMemset(d_err, 0, 8));
    if (s->n_series) k_fill_seg_series<<<s->n_series, 128>>>(s->d_series_seg_begin, s->n_series, s->d_seg_series);
    if (s->n_segments && scan_snappy) { /* Snappy pages -> raw pages appended behind the data (snappy_load.cuh) */
        const size_t n_pages = (size_t)(s->n_columns + 1) * s->n_segments;
        Scratch tr;
        uint32_t *tr_size; unsigned long long *d_cnt;
        if ((rc = tr.get(&tr_size, n_pages)) || (rc = tr.get(&d_cnt, 3))) return rc;
        CU(cudaMemset(d_cnt, 0, 24));
        k_snappy_scan<<<(s->n_segments + 127) / 128, 128>>>(make_dir(s), d_types, tr_size, d_cnt);
        unsigned long long cnt[3];
        CU(cudaMemcpy(cnt, d_cnt, 24, cudaMemcpyDeviceToHost));
        if (cnt[0]) {
            if (!s->owns_data) { set_error("shard has %llu Snappy pages: they are transcoded at open, which needs a library-owned copy of the data (do not pass OG_SHARD_DEVICE_DATA)", cnt[0]); return OG_E_UNSUPPORTED; }
            uint64_t *tr_off; uint8_t *scan_tmp; size_t tb = 0;
            if ((rc = tr.get(&tr_off, n_pages))) return rc;
            CU(cub::DeviceScan::ExclusiveSum(nullptr, tb, tr_size, tr_off, (int)n_pages));
            if ((rc = tr.get(&scan_tmp, tb))) return rc;
            CU(cub::DeviceScan::ExclusiveSum(scan_tmp, tb, tr_size, tr_off, (int)n_pages));
            const uint64_t new_base = (s->data_len + 15) & ~15ull, new_len = new_base + cnt[2];
            /* the shard takes the new buffer at once; the loaded pages stay readable until `tr` releases them */
            const DirP loaded = make_dir(s);
            uint8_t *nd;
            if ((rc = dalloc(&nd, (size_t)new_len + 1024))) return rc;
            tr.bufs.push_back(s->d_data); s->d_data = nd;
            CU(cudaMemcpy(nd, loaded.data, s->data_len, cudaMemcpyDeviceToDevice));
            CU(cudaMemset(nd + s->data_len, 0, new_len + 1024 - s->data_len));
            k_snappy_transcode<<<(unsigned)((n_pages + 127) / 128), 128>>>(loaded, tr_size, tr_off, nd, new_base, s->d_page_off, s->d_page_len, d_err);
            CU(cudaGetLastError());
            CU(cudaDeviceSynchronize());
            s->data_len = new_len;
            s->snappy_pages = cnt[0]; s->snappy_bytes_in = cnt[1]; s->snappy_bytes_out = cnt[2];
        }
    }
    if (s->n_segments) k_validate<<<(s->n_segments + 127) / 128, 128>>>(make_dir(s), d_types, s->d_seg_rows, d_tot, d_max, d_err);
    CU(cudaGetLastError());
    unsigned long long tot[3]; int err[2]; uint32_t mx;
    CU(cudaMemcpy(tot, d_tot, 24, cudaMemcpyDeviceToHost));
    CU(cudaMemcpy(err, d_err, 8, cudaMemcpyDeviceToHost));
    CU(cudaMemcpy(&mx, d_max, 4, cudaMemcpyDeviceToHost));
    if (err[0]) {
        set_error("segment %d: %s page (device validation code %d)", err[1], err[0] == D_UNSUPPORTED ? "unsupported codec in" : err[0] == D_TYPE ? "type mismatch in" : "corrupt", err[0]);
        return map_dev_err(err[0]);
    }
    s->n_rows = tot[0]; s->page_bytes = tot[1] - s->snappy_bytes_out + s->snappy_bytes_in; /* algorithmic bytes = the pages as the files stored them (ogpu.h og_shard_info) */
    s->max_seg_rows = mx; s->irregular_time_pages = tot[2];
    return OG_OK;
}

/* the six directory arrays of a shard whose n_series, n_segments and n_columns are set */
int alloc_dir(og_shard *s) {
    const size_t nseg = s->n_segments, n_pages = ((size_t)s->n_columns + 1) * nseg;
    int rc;
    if ((rc = dalloc(&s->d_series_seg_begin, (size_t)s->n_series + 1)) || (rc = dalloc(&s->d_tmin, nseg)) || (rc = dalloc(&s->d_tmax, nseg)) ||
        (rc = dalloc(&s->d_page_off, n_pages)) || (rc = dalloc(&s->d_page_len, n_pages)) || (rc = dalloc(&s->d_sids, (size_t)s->n_series)))
        return rc;
    return OG_OK;
}

/* ... allocated and filled from host arrays of those sizes (page_off / page_len column-major, time column last) */
int upload_dir(og_shard *s, const uint32_t *series_seg_begin, const int64_t *seg_tmin, const int64_t *seg_tmax, const uint64_t *page_off,
               const uint32_t *page_len, const uint64_t *sids) {
    int rc = alloc_dir(s); if (rc) return rc;
    const size_t nseg = s->n_segments, n_pages = ((size_t)s->n_columns + 1) * nseg;
    CU(cudaMemcpy(s->d_series_seg_begin, series_seg_begin, ((size_t)s->n_series + 1) * 4, cudaMemcpyHostToDevice));
    CU(cudaMemcpy(s->d_tmin, seg_tmin, nseg * 8, cudaMemcpyHostToDevice));
    CU(cudaMemcpy(s->d_tmax, seg_tmax, nseg * 8, cudaMemcpyHostToDevice));
    CU(cudaMemcpy(s->d_page_off, page_off, n_pages * 8, cudaMemcpyHostToDevice));
    CU(cudaMemcpy(s->d_page_len, page_len, n_pages * 4, cudaMemcpyHostToDevice));
    CU(cudaMemcpy(s->d_sids, sids, (size_t)s->n_series * 8, cudaMemcpyHostToDevice));
    return OG_OK;
}

} // namespace ogpu

using namespace ogpu;

/* =============================================== lifecycle =============================================== */
extern "C" {

OG_API int og_device_count(void) { int n = 0; if (cudaGetDeviceCount(&n) != cudaSuccess) return 0; return n; }

OG_API int og_init(int device_ordinal) {
    int n = og_device_count();
    if (n <= 0) { set_error("no CUDA device visible: libogpu has no CPU path"); return OG_E_CUDA; }
    if (device_ordinal < 0 || device_ordinal >= n) { set_error("device ordinal %d out of range (%d devices)", device_ordinal, n); return OG_E_INVAL; }
    CU(cudaSetDevice(device_ordinal));
    CU(cudaFree(0));
    { /* keep freed buffers in the device's memory pool (see internal.h dev_malloc) */
        cudaMemPool_t pool; uint64_t thr = ~0ull;
        if (cudaDeviceGetDefaultMemPool(&pool, device_ordinal) == cudaSuccess) cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &thr);
        else cudaGetLastError();
    }
    g_device = device_ordinal;
    return OG_OK;
}

OG_API const char *og_strerror(int st) {
    switch (st) {
    case OG_OK: return "ok";
    case OG_EOF: return "end of stream";
    case OG_E_INVAL: return "invalid argument";
    case OG_E_CUDA: return "CUDA failure or no device bound";
    case OG_E_NOMEM: return "out of device memory";
    case OG_E_UNSUPPORTED: return "unsupported codec or option on the GPU path";
    case OG_E_CORRUPT: return "corrupt page";
    case OG_E_ABORTED: return "query aborted";
    case OG_E_TYPE: return "column type mismatch";
    case OG_E_STATE: return "call sequence error";
    default: return "unknown status";
    }
}
OG_API const char *og_last_error(void) { return g_err; }
OG_API const char *og_version(void) { return "ogpu 0.2 (sm_90a)"; }
OG_API int og_release_cached_memory(void) {
    if (g_device < 0) return OG_OK;
    CU(cudaSetDevice(g_device));
    CU(cudaDeviceSynchronize());
    cudaMemPool_t pool;
    CU(cudaDeviceGetDefaultMemPool(&pool, g_device));
    CU(cudaMemPoolTrimTo(pool, 0));
    return OG_OK;
}

/* =============================================== shard =============================================== */
} // extern "C"
namespace ogpu {
int ensure_device() {
    if (g_device < 0) { int rc = og_init(0); if (rc != OG_OK) return rc; }
    else CU(cudaSetDevice(g_device));
    return OG_OK;
}
} // namespace ogpu
static int need_device() { return ogpu::ensure_device(); }
extern "C" {

OG_API void og_shard_close(og_shard *s) { delete s; }

} // extern "C"
namespace ogpu {
/* host checks of one shard description: og_shard_open and og_shard_open_files (merge.cu) run them on every description */
int check_desc(const og_shard_desc *d) {
    if (d->n_columns > 64 || (d->n_segments && (!d->seg_tmin || !d->seg_tmax || !d->time_page_off || !d->time_page_len)) || (d->n_series && !d->series_seg_begin)) { set_error("bad shard descriptor"); return OG_E_INVAL; }
    for (uint32_t s = 0; s < d->n_series; s++) if (d->series_seg_begin[s] > d->series_seg_begin[s + 1]) { set_error("series_seg_begin not monotone at %u", s); return OG_E_INVAL; }
    if (d->n_series && d->series_seg_begin[d->n_series] != d->n_segments) { set_error("series_seg_begin[n_series] != n_segments"); return OG_E_INVAL; }
    for (uint32_t c = 0; c < d->n_columns; c++)
        if (d->columns[c].type != OG_TYPE_INT && d->columns[c].type != OG_TYPE_FLOAT && d->columns[c].type != OG_TYPE_BOOL && d->columns[c].type != OG_TYPE_STRING) {
            set_error("column %u: unknown column type %d", c, d->columns[c].type); return OG_E_UNSUPPORTED;
        }
    for (size_t c = 0; c <= d->n_columns; c++) {
        const uint64_t *po = c < d->n_columns ? d->columns[c].page_off : d->time_page_off;
        const uint32_t *pl = c < d->n_columns ? d->columns[c].page_len : d->time_page_len;
        for (size_t g = 0; g < d->n_segments; g++)
            if (po[g] + pl[g] > d->data_len) { set_error("column %zu segment %zu: page [%llu,+%u) outside data (%llu bytes)", c, g, (unsigned long long)po[g], pl[g], (unsigned long long)d->data_len); return OG_E_INVAL; }
    }
    for (uint32_t sr = 0; sr < d->n_series; sr++)
        for (uint32_t g = d->series_seg_begin[sr]; g < d->series_seg_begin[sr + 1]; g++)
            if (d->seg_tmin[g] > d->seg_tmax[g] || (g > d->series_seg_begin[sr] && d->seg_tmin[g] <= d->seg_tmax[g - 1])) {
                set_error("series %u: segment %u is not time-ordered (only ordered TSSP files are supported)", sr, g); return OG_E_UNSUPPORTED;
            }
    return OG_OK;
}
} // namespace ogpu
extern "C" {

OG_API int og_shard_open(const og_shard_desc *d, og_shard **out) {
    if (!d || !out) { set_error("null argument"); return OG_E_INVAL; }
    *out = nullptr;
    int rc = need_device(); if (rc) return rc;
    if ((rc = check_desc(d))) return rc;
    std::unique_ptr<og_shard> s(new og_shard);
    s->device = g_device; s->n_series = d->n_series; s->n_segments = d->n_segments; s->n_columns = d->n_columns;
    s->data_len = d->data_len;
    for (uint32_t c = 0; c < d->n_columns; c++) {
        s->col_types.push_back(d->columns[c].type);
        s->col_names.push_back(d->columns[c].name ? d->columns[c].name : "");
    }
    s->sids.assign(d->sids, d->sids + d->n_series);
    s->h_series_seg_begin.assign(d->series_seg_begin, d->series_seg_begin + d->n_series + 1);
    size_t nseg = d->n_segments, ncol1 = (size_t)d->n_columns + 1;
    std::vector<uint64_t> off(ncol1 * nseg); std::vector<uint32_t> len(ncol1 * nseg);
    for (size_t c = 0; c < ncol1; c++) {
        const uint64_t *po = c < d->n_columns ? d->columns[c].page_off : d->time_page_off;
        const uint32_t *pl = c < d->n_columns ? d->columns[c].page_len : d->time_page_len;
        for (size_t g = 0; g < nseg; g++) { off[c * nseg + g] = po[g]; len[c * nseg + g] = pl[g]; }
    }
    s->tmin = INT64_MAX; s->tmax = INT64_MIN;
    if (d->n_series)
        for (uint32_t g = d->series_seg_begin[0]; g < d->series_seg_begin[d->n_series]; g++) { s->tmin = std::min(s->tmin, d->seg_tmin[g]); s->tmax = std::max(s->tmax, d->seg_tmax[g]); }
    if (d->flags & OG_SHARD_DEVICE_DATA) { s->d_data = (uint8_t *)d->data; s->owns_data = false; }
    else {
        if ((rc = dalloc(&s->d_data, d->data_len + 1024))) return rc; /* tail padding: word-wise unaligned loads and the interleave repack read past the last page */
        CU(cudaMemcpy(s->d_data, d->data, d->data_len, cudaMemcpyHostToDevice));
        CU(cudaMemset(s->d_data + d->data_len, 0, 1024));
    }
    if ((rc = upload_dir(s.get(), d->series_seg_begin, d->seg_tmin, d->seg_tmax, off.data(), len.data(), d->sids))) return rc;
    if ((rc = shard_finalize(s.get(), true))) return rc;
    *out = s.release();
    return OG_OK;
}

OG_API int og_shard_info(const og_shard *s, uint64_t *n_series, uint64_t *n_segments, uint64_t *n_rows, uint64_t *page_bytes, int64_t *tmin, int64_t *tmax) {
    if (!s) return OG_E_INVAL;
    if (n_series) *n_series = s->n_series;
    if (n_segments) *n_segments = s->n_segments;
    if (n_rows) *n_rows = s->n_rows;
    if (page_bytes) *page_bytes = s->page_bytes;
    if (tmin) *tmin = s->tmin;
    if (tmax) *tmax = s->tmax;
    return OG_OK;
}

OG_API int og_shard_layout_get(const og_shard *s, og_shard_layout *out) {
    if (!s || !out) return OG_E_INVAL;
    out->data_len = s->data_len; out->n_series = s->n_series; out->n_segments = s->n_segments; out->n_columns = s->n_columns;
    return OG_OK;
}

OG_API int og_shard_export(const og_shard *s, uint8_t *data, uint64_t *sids, uint32_t *series_seg_begin, int64_t *seg_tmin,
                           int64_t *seg_tmax, uint64_t *page_off, uint32_t *page_len, int32_t *col_types) {
    if (!s) return OG_E_INVAL;
    CU(cudaSetDevice(s->device));
    size_t nseg = s->n_segments, ncol1 = (size_t)s->n_columns + 1;
    if (data) CU(cudaMemcpy(data, s->d_data, s->data_len, cudaMemcpyDeviceToHost));
    if (sids) memcpy(sids, s->sids.data(), s->sids.size() * 8);
    if (series_seg_begin) memcpy(series_seg_begin, s->h_series_seg_begin.data(), s->h_series_seg_begin.size() * 4);
    if (seg_tmin) CU(cudaMemcpy(seg_tmin, s->d_tmin, nseg * 8, cudaMemcpyDeviceToHost));
    if (seg_tmax) CU(cudaMemcpy(seg_tmax, s->d_tmax, nseg * 8, cudaMemcpyDeviceToHost));
    if (page_off) CU(cudaMemcpy(page_off, s->d_page_off, ncol1 * nseg * 8, cudaMemcpyDeviceToHost));
    if (page_len) CU(cudaMemcpy(page_len, s->d_page_len, ncol1 * nseg * 4, cudaMemcpyDeviceToHost));
    if (col_types) memcpy(col_types, s->col_types.data(), s->col_types.size() * 4);
    return OG_OK;
}

/* =============================================== query =============================================== */
static const int64_t MIN_TIME = INT64_MIN + 2, MAX_TIME = INT64_MAX - 1;
/* ProcessorOptions.Window (lib/util/lifted/influx/query/select.go:579-655, Location == nil); host-side only:
 * the kernels use the affine form start + b*interval that it implies for in-range rows. */
static void window_of(int64_t interval, int64_t offset, int64_t tmin, int64_t tmax, int64_t t, int64_t *s, int64_t *e) {
    if (interval == 0) { *s = tmin; *e = tmax + 1; return; }
    t -= offset;
    int64_t dt = t % interval;
    if (dt < 0) dt += interval;
    int64_t st = ((int64_t)((uint64_t)MIN_TIME + (uint64_t)dt) >= t) ? MIN_TIME : t - dt;
    st += offset;
    int64_t d2 = interval - dt;
    int64_t en = (MAX_TIME - d2 <= t) ? MAX_TIME : t + d2;
    en += offset;
    *s = st; *e = en;
}
/* Window() clamps the window of t at MIN_TIME or MAX_TIME when the aligned window would reach past them.  The kernels place
 * row t in bucket (t - start) / interval, which holds only on the unclamped grid, so og_query_create refuses a range whose
 * first or last row lies in a clamped window (DESIGN.md "Deviations").  The window after the last row may be clamped: it
 * only sets the bucket count, and every row still has its bucket. */
static bool window_clamped(int64_t interval, int64_t offset, int64_t t) {
    const __int128 x = (__int128)t - offset;
    __int128 r = x % interval;
    if (r < 0) r += interval;
    const __int128 s = x - r, e = s + interval;
    return s < MIN_TIME || e > MAX_TIME || s + offset < INT64_MIN || e + offset > INT64_MAX;
}

} /* extern "C" */
namespace { void free_plan(void *plan); }
extern "C" void og_query_free_merge_state(void *p);
/* callers may still have work enqueued on the stream (og_dense_view.stream) that reads the dense record: wait for it */
og_query::~og_query() {
    if (stream) cudaStreamSynchronize(stream);
    if (live) { std::lock_guard<std::mutex> lock(live->mu); live->n--; }
    og_query_free_merge_state(merge_state);
    free_plan(plan);
    if (ev0) cudaEventDestroy(ev0);
    if (ev1) cudaEventDestroy(ev1);
    for (cudaEvent_t e : main_ev) cudaEventDestroy(e);
    if (stream) cudaStreamDestroy(stream);
}
extern "C" {
OG_API void og_query_destroy(og_query *q) { delete q; }

OG_API int og_query_create(og_shard *s, const og_query_desc *d_in, og_query **out) {
    if (!s || !d_in || !out) { set_error("null argument"); return OG_E_INVAL; }
    *out = nullptr;
    /* influxql.MinTime/MaxTime (ast.go:92,102) bound every query range, so that EndTime+1 in Window() cannot overflow */
    og_query_desc d_clamped = *d_in;
    d_clamped.tmin = std::max(d_in->tmin, MIN_TIME); d_clamped.tmax = std::min(d_in->tmax, MAX_TIME);
    const og_query_desc *d = &d_clamped;
    CU(cudaSetDevice(s->device));
    /* ascending == 0 (ORDER BY time DESC): the windows and their aggregates are computed exactly as for an ascending scan and
     * og_query_next emits the rows of every group from the latest window to the earliest.  Where the reference's reversed-record
     * reduction could differ — which of two equal extremes inside one window lends its time to a single-call min/max, the
     * association of float sums — the ascending rules apply (float sums stay within the 1e-9 bound; see DESIGN.md). */
    if (d->n_calls == 0 || d->n_calls > OG_MAX_CALLS) { set_error("n_calls must be 1..%d", OG_MAX_CALLS); return OG_E_INVAL; }
    if (d->n_filter > OG_MAX_FILTER) { set_error("filter too long (max %d items)", OG_MAX_FILTER); return OG_E_INVAL; }
    if (d->interval < 0 || d->tmin > d->tmax) { set_error("bad interval or time range"); return OG_E_INVAL; }
    std::unique_ptr<og_query> q(new og_query);
    { /* waits while og_shard_append_files runs on the shard */
        std::lock_guard<std::mutex> lock(s->live->mu);
        s->live->n++;
        q->sh = s; q->live = s->live;
    }
    q->desc = *d;
    q->calls.assign(d->calls, d->calls + d->n_calls);
    if (d->n_filter) q->filter.assign(d->filter, d->filter + d->n_filter);
    q->desc.calls = q->calls.data(); q->desc.filter = q->filter.data();
    QueryP &p = q->qp;
    memset(&p, 0, sizeof p);
    /* column slots */
    auto slot_of = [&](int col) -> int {
        for (uint32_t i = 0; i < p.n_cols; i++) if (p.col_index[i] == col) return (int)i;
        if (p.n_cols >= OG_MAX_COLS) return -1;
        p.col_index[p.n_cols] = col; p.col_type[p.n_cols] = s->col_types[col];
        return (int)p.n_cols++;
    };
    for (uint32_t i = 0; i < d->n_calls; i++) {
        const og_call &c = d->calls[i];
        if (c.column < 0 || (uint32_t)c.column >= s->n_columns || c.func < OG_AGG_COUNT || c.func > OG_AGG_LAST) { set_error("call %u: bad column or function", i); return OG_E_INVAL; }
        int type = s->col_types[c.column];
        if (type == OG_TYPE_STRING && c.func != OG_AGG_COUNT) { set_error("call %u: only count() is pushed down for string columns (their values are never decoded on the GPU path)", i); return OG_E_UNSUPPORTED; }
        if (c.func == OG_AGG_SUM && type == OG_TYPE_BOOL) { set_error("sum() over a boolean column (unsupported sum iterator type, series_call_processor.go:140)"); return OG_E_INVAL; }
        int sl = slot_of(c.column);
        if (sl < 0) { set_error("too many distinct columns"); return OG_E_INVAL; }
        p.calls[i].func = c.func; p.calls[i].col_slot = sl; p.calls[i].type = type;
        p.calls[i].out_type = c.func == OG_AGG_COUNT ? OG_TYPE_INT : type;
    }
    p.n_calls = d->n_calls; p.multi = d->n_calls > 1;
    int sp = 0;
    for (uint32_t i = 0; i < d->n_filter; i++) {
        const og_filter_item &f = d->filter[i];
        FilterP &fp = p.filter[i];
        fp.kind = f.kind;
        if (f.kind == OG_F_TERM) {
            if (f.column < 0 || (uint32_t)f.column >= s->n_columns || f.op < OG_OP_LT || f.op > OG_OP_NEQ) { set_error("filter item %u: bad column or op", i); return OG_E_INVAL; }
            if (s->col_types[f.column] == OG_TYPE_STRING) { set_error("filter item %u: WHERE on a string column is not pushed down", i); return OG_E_UNSUPPORTED; }
            int sl = slot_of(f.column);
            if (sl < 0) { set_error("too many distinct columns"); return OG_E_INVAL; }
            fp.col_slot = sl; fp.op = f.op; fp.type = s->col_types[f.column]; fp.const_is_float = f.const_is_float; fp.fval = f.fval; fp.ival = f.ival;
            sp++;
        } else if (f.kind == OG_F_AND || f.kind == OG_F_OR) {
            if (sp < 2) { set_error("filter RPN underflow at item %u", i); return OG_E_INVAL; }
            sp--;
        } else { set_error("filter item %u: bad kind", i); return OG_E_INVAL; }
    }
    if (d->n_filter && sp != 1) { set_error("filter RPN does not reduce to one value"); return OG_E_INVAL; }
    p.n_filter = d->n_filter;
    /* bucket geometry: TimeWindowsInit (agg_tagset_cursor.go:1012-1027) over the query range (updateQueryTime :448-463) */
    /* FileInfo.{Min,Max}Time is the file range intersected with the query range (fileLoopCursor.updateQueryTime :448-463),
     * so open-ended queries (opt.StartTime/EndTime = Min/MaxTime) get a bounded interval record. */
    int64_t gmin = std::max(d->tmin, s->tmin), gmax = std::min(d->tmax, s->tmax);
    bool overlap = gmin <= gmax;
    if (!overlap) gmin = gmax = d->tmin; /* no overlap: one empty window */
    if (d->flags & OG_Q_QUERY_GRID) { /* one grid for every shard of a cross-shard query */
        if (d_in->tmin <= MIN_TIME || d_in->tmax >= MAX_TIME) { set_error("OG_Q_QUERY_GRID needs a bounded time range"); return OG_E_INVAL; }
        gmin = d->tmin; gmax = d->tmax; overlap = true;
    }
    int64_t s0, e0, s1, e1;
    if (d->interval == 0) { s0 = gmin; e0 = gmax + 1; s1 = s0; e1 = e0; }
    else {
        /* (a range without rows keeps its one empty window, clamped or not: nothing is placed in it) */
        if (overlap && (window_clamped(d->interval, d->offset, gmin) || window_clamped(d->interval, d->offset, gmax))) {
            set_error("the first or last window of the range is clamped at the int64 time limits"); return OG_E_UNSUPPORTED;
        }
        window_of(d->interval, d->offset, d->tmin, d->tmax, gmin, &s0, &e0);
        window_of(d->interval, d->offset, d->tmin, d->tmax, gmax + 1, &s1, &e1);
    }
    p.tmin = d->tmin; p.tmax = d->tmax; p.start = s0; p.interval = e0 - s0;
    if (p.interval <= 0) { set_error("degenerate window"); return OG_E_INVAL; }
    uint64_t nb = d->interval ? (uint64_t)(e1 - s0) / (uint64_t)p.interval : 1;
    if (nb == 0 || nb > 0x7fffffffull) { set_error("query range yields %llu buckets", (unsigned long long)nb); return OG_E_INVAL; }
    p.n_buckets = (uint32_t)nb;
    /* groups */
    q->n_groups = d->group_mode == OG_GROUP_ALL ? 1 : d->group_mode == OG_GROUP_PER_SERIES ? s->n_series : d->n_groups;
    if (d->group_mode == OG_GROUP_MAP) {
        if (!d->series_group || d->n_groups == 0) { set_error("OG_GROUP_MAP needs series_group and n_groups"); return OG_E_INVAL; }
        q->series_group.assign(d->series_group, d->series_group + s->n_series);
        for (uint32_t g : q->series_group) if (g >= d->n_groups) { set_error("series_group entry out of range"); return OG_E_INVAL; }
    } else if (d->group_mode != OG_GROUP_ALL && d->group_mode != OG_GROUP_PER_SERIES) { set_error("bad group_mode"); return OG_E_INVAL; }
    if (q->n_groups == 0) q->n_groups = 1;
    cudaError_t e = cudaStreamCreateWithFlags(&q->stream, cudaStreamNonBlocking);
    if (e != cudaSuccess) return cuda_fail(e, "cudaStreamCreate", __FILE__, __LINE__);
    cudaEventCreate(&q->ev0); cudaEventCreate(&q->ev1);
    *out = q.release();
    return OG_OK;
}

OG_API void og_query_abort(og_query *q) { if (q) q->aborted = 1; }

} /* extern "C" */
namespace {
struct Plan { /* built once per query, reused by every og_query_run */
    ChunkP ch; TileP tp; GroupP gp;
    bool fused;
    bool cols;      /* multi, served by the column-at-a-time kernel k_fused_cols */
    bool multi;     /* several columns and/or a WHERE: pull-iterator kernel k_fused_multi, nothing materialised */
    bool fast;      /* the fused Gorilla kernel serves the eligible segments, k_fused_segment the rest */
    bool blockmerge;/* one tagset, order not pinned, per-series cells: two-stage parallel merge (k_merge_all_blocks + k_merge_folded) */
    bool fold;      /* interior windows are folded in-warp into gcells (one tagset, regular shard, no strict order) */
    int fm; bool times;
    IlP il;
    const og_shard::IlCol *ic;
};
void free_plan(void *plan) { delete (Plan *)plan; }

template <int NC> void launch_fused(const DirP &d, const QueryP &p, const ChunkP &ch, const uint32_t *list, uint32_t n, cudaStream_t st) {
    if (n) k_fused_segment<NC><<<(n + 127) / 128, 128, 0, st>>>(d, p, ch, list, n);
}
template <int FM, bool TIMES> void launch_fast_t(bool fold, const IlP &il, uint32_t g0, uint32_t g1, const QueryP &p, const ChunkP &ch, cudaStream_t st) {
    constexpr uint32_t WPB = OG_FAST_THREADS / 32;
    dim3 grid((g1 - g0 + WPB - 1) / WPB), block(OG_FAST_THREADS);
    if (fold) k_fused_il<FM, TIMES, true><<<grid, block, WPB * il_acc_bytes(p.n_calls, TIMES), st>>>(p, ch, il, g0, g1);
    else k_fused_il<FM, TIMES, false><<<grid, block, 0, st>>>(p, ch, il, g0, g1);
}
/* a handful of aggregate-set specialisations; anything else runs the all-aggregates instance */
void launch_fast(int fm, bool times, bool fold, const IlP &il, uint32_t g0, uint32_t g1, const QueryP &p, const ChunkP &ch, cudaStream_t st) {
    if (g1 <= g0) return;
    if (!times) {
        switch (fm) {
        case FM_SUM | FM_COUNT: return launch_fast_t<FM_SUM | FM_COUNT, false>(fold, il, g0, g1, p, ch, st);
        case FM_SUM | FM_COUNT | FM_MAX: return launch_fast_t<FM_SUM | FM_COUNT | FM_MAX, false>(fold, il, g0, g1, p, ch, st);
        case FM_SUM | FM_COUNT | FM_MIN | FM_MAX: return launch_fast_t<FM_SUM | FM_COUNT | FM_MIN | FM_MAX, false>(fold, il, g0, g1, p, ch, st);
        case FM_COUNT: return launch_fast_t<FM_COUNT, false>(fold, il, g0, g1, p, ch, st);
        default: break;
        }
    } else {
        switch (fm) {
        case FM_MAX | FM_COUNT: return launch_fast_t<FM_MAX | FM_COUNT, true>(fold, il, g0, g1, p, ch, st);
        case FM_MIN | FM_COUNT: return launch_fast_t<FM_MIN | FM_COUNT, true>(fold, il, g0, g1, p, ch, st);
        default: break;
        }
    }
    return launch_fast_t<63, true>(fold, il, g0, g1, p, ch, st);
}

template <int NCOL, int NCALL> void launch_multi_t(const QueryP &p, const DirP &d, const ChunkP &ch, uint32_t nseg, cudaStream_t st) {
    bool simple = true;
    for (uint32_t c = 0; c < p.n_calls; c++) simple &= p.calls[c].func == OG_AGG_COUNT || p.calls[c].func == OG_AGG_SUM;
    const unsigned gb = (nseg + 127) / 128;
    if (simple) k_fused_multi<NCOL, NCALL, true><<<gb, 128, 0, st>>>(d, p, ch);
    else k_fused_multi<NCOL, NCALL, false><<<gb, 128, 0, st>>>(d, p, ch);
}
template <int NCOL> void launch_multi_c(const QueryP &p, const DirP &d, const ChunkP &ch, uint32_t nseg, cudaStream_t st) {
    switch (p.n_calls) {
    case 1: return launch_multi_t<NCOL, 1>(p, d, ch, nseg, st);
    case 2: return launch_multi_t<NCOL, 2>(p, d, ch, nseg, st);
    case 3: return launch_multi_t<NCOL, 3>(p, d, ch, nseg, st);
    case 4: return launch_multi_t<NCOL, 4>(p, d, ch, nseg, st);
    case 5: return launch_multi_t<NCOL, 5>(p, d, ch, nseg, st);
    case 6: return launch_multi_t<NCOL, 6>(p, d, ch, nseg, st);
    case 7: return launch_multi_t<NCOL, 7>(p, d, ch, nseg, st);
    default: return launch_multi_t<NCOL, 8>(p, d, ch, nseg, st);
    }
}
void launch_cols(const QueryP &p, const DirP &d, const ChunkP &ch, uint32_t nseg, cudaStream_t st) {
    bool simple = true;
    for (uint32_t c = 0; c < p.n_calls; c++) simple &= p.calls[c].func == OG_AGG_COUNT || p.calls[c].func == OG_AGG_SUM;
    const unsigned gb = (nseg + 127) / 128;
    if (simple) k_fused_cols<true><<<gb, 128, 0, st>>>(d, p, ch);
    else k_fused_cols<false><<<gb, 128, 0, st>>>(d, p, ch);
}
void launch_multi(const QueryP &p, const DirP &d, const ChunkP &ch, uint32_t nseg, cudaStream_t st) {
    switch (p.n_cols) {
    case 1: return launch_multi_c<1>(p, d, ch, nseg, st);
    case 2: return launch_multi_c<2>(p, d, ch, nseg, st);
    case 3: return launch_multi_c<3>(p, d, ch, nseg, st);
#ifdef OG_WIDE_MULTI
    case 5: return launch_multi_c<5>(p, d, ch, nseg, st);
    case 6: return launch_multi_c<6>(p, d, ch, nseg, st);
    case 7: return launch_multi_c<7>(p, d, ch, nseg, st);
    case 8: return launch_multi_c<8>(p, d, ch, nseg, st);
#endif
    default: return launch_multi_c<4>(p, d, ch, nseg, st);
    }
}

/* Build (once per shard and column) the lane-interleaved, length-binned stream copy that k_fused_il reads (il_build.cuh).
 * Returns OG_OK with state 1 (ready), -1 (nothing eligible) or -2 (not enough device memory: the general fused kernel
 * serves the column instead; visible in og_stats.il_state). */
int ensure_il(og_shard *s, int col, cudaStream_t st) {
    std::lock_guard<std::mutex> lock(s->il_mu);
    if (s->il.size() != s->n_columns) s->il.resize(s->n_columns);
    og_shard::IlCol &ic = s->il[col];
    if (ic.state != 0) return OG_OK;
    ic.state = -1;
    if (s->n_segments == 0 || s->col_types[col] != OG_TYPE_FLOAT) return OG_OK;
    const uint32_t nseg = s->n_segments;
    /* regular shard: every series has the same number of segments -> lane groups share a segment index */
    uint32_t J = s->n_series ? s->h_series_seg_begin[1] - s->h_series_seg_begin[0] : 0;
    for (uint32_t i = 0; i < s->n_series && J; i++) if (s->h_series_seg_begin[i + 1] - s->h_series_seg_begin[i] != J) J = 0;
    const uint32_t n_super = J ? (s->n_series + OG_IL_SUPER - 1) / OG_IL_SUPER : 1;
    const uint64_t n_dom64 = J ? (uint64_t)n_super * J : 1;
    if (n_dom64 >= (1ull << 31)) return OG_OK;
    const uint32_t n_dom = (uint32_t)n_dom64;
    int rc;
    EventTimer timer(st);
    timer.start();
    Scratch tmp(st); /* k_il_scan and the sort may still run on st when a check below returns */
    IlScanOut so{};
    uint32_t *seg_words; uint64_t *keys2; uint32_t *vals2;
    if ((rc = tmp.get(&so.seg_win, nseg)) || (rc = tmp.get(&so.n_packed, 1)) ||
        (rc = tmp.get(&seg_words, nseg)) || (rc = tmp.get(&so.seg_t0, nseg)) || (rc = tmp.get(&so.seg_dt, nseg)) || (rc = tmp.get(&so.keys, nseg)) ||
        (rc = tmp.get(&so.vals, nseg)) || (rc = tmp.get(&keys2, nseg)) || (rc = tmp.get(&vals2, nseg)) || (rc = tmp.get(&so.dom_cnt, n_dom))) return rc;
    so.seg_words = seg_words;
    if ((rc = tmp.get(&so.misaligned, 1))) return rc;
    CU(cudaMemsetAsync(so.dom_cnt, 0, (size_t)n_dom * 4, st));
    CU(cudaMemsetAsync(so.misaligned, 0, 4, st));
    CU(cudaMemsetAsync(so.n_packed, 0, 8, st));
    DirP d = make_dir(s);
    k_il_scan<<<(nseg + 255) / 256, 256, 0, st>>>(d, col, s->col_types[col], J, so);
    CU(cudaGetLastError());
    /* stable sort by (domain, words): not-eligible segments (key ~0) end up last, in segment order */
    int dbits = 1; while ((1ull << dbits) < n_dom64 + 1) dbits++;
    {
        size_t tb = 0;
        CU(cub::DeviceRadixSort::SortPairs(nullptr, tb, so.keys, keys2, so.vals, vals2, (int)nseg, 0, (int)OG_IL_WORD_BITS + dbits, st));
        void *dtmp; if ((rc = tmp.get((uint8_t **)&dtmp, tb))) return rc;
        CU(cub::DeviceRadixSort::SortPairs(dtmp, tb, so.keys, keys2, so.vals, vals2, (int)nseg, 0, (int)OG_IL_WORD_BITS + dbits, st));
    }
    std::vector<uint32_t> dom_cnt(n_dom); uint32_t misaligned = 1; unsigned long long n_packed = 0;
    CU(cudaMemcpyAsync(dom_cnt.data(), so.dom_cnt, (size_t)n_dom * 4, cudaMemcpyDeviceToHost, st));
    CU(cudaMemcpyAsync(&misaligned, so.misaligned, 4, cudaMemcpyDeviceToHost, st));
    CU(cudaMemcpyAsync(&n_packed, so.n_packed, 8, cudaMemcpyDeviceToHost, st));
    CU(cudaStreamSynchronize(st));
    std::vector<uint32_t> elem_first(n_dom), grp_first(n_dom);
    uint64_t n_elig = 0, ng64 = 0;
    for (uint32_t i = 0; i < n_dom; i++) { elem_first[i] = (uint32_t)n_elig; grp_first[i] = (uint32_t)ng64; n_elig += dom_cnt[i]; ng64 += (dom_cnt[i] + 31) / 32; }
    /* the segments the fused kernel does not take: the tail of the sorted order */
    const uint32_t n_gen = nseg - (uint32_t)n_elig;
    if (n_gen) {
        if ((rc = dalloc(&ic.gen_list, (size_t)n_gen))) return rc;
        CU(cudaMemcpyAsync(ic.gen_list, vals2 + n_elig, (size_t)n_gen * 4, cudaMemcpyDeviceToDevice, st));
        ic.gen_host.resize(n_gen);
        CU(cudaMemcpyAsync(ic.gen_host.data(), vals2 + n_elig, (size_t)n_gen * 4, cudaMemcpyDeviceToHost, st));
        CU(cudaStreamSynchronize(st));
    }
    if (n_elig == 0) return OG_OK;
    const uint32_t ng = (uint32_t)ng64;
    ic.n_groups = ng; ic.J = J; ic.aligned = J != 0 && misaligned == 0; ic.n_super = n_super; ic.cols_per_super = OG_IL_SUPER / 32 + 1;
    ic.super_grp_first.assign(n_super + 1, ng);
    for (uint32_t sp = 0; sp < n_super; sp++) ic.super_grp_first[sp] = grp_first[J ? sp * J : 0];
    uint32_t *d_elem_first, *d_grp_first;
    if ((rc = tmp.get(&d_elem_first, n_dom)) || (rc = tmp.get(&d_grp_first, n_dom))) return rc;
    CU(cudaMemcpyAsync(d_elem_first, elem_first.data(), (size_t)n_dom * 4, cudaMemcpyHostToDevice, st));
    CU(cudaMemcpyAsync(d_grp_first, grp_first.data(), (size_t)n_dom * 4, cudaMemcpyHostToDevice, st));
    const size_t n_slots = (size_t)ng * 32;
    if ((rc = dalloc(&ic.lane_seg, n_slots)) || (rc = dalloc(&ic.lane_rows, n_slots)) || (rc = dalloc(&ic.lane_win, n_slots)) || (rc = dalloc(&ic.lane_series, n_slots)) ||
        (rc = dalloc(&ic.lane_t0, n_slots)) || (rc = dalloc(&ic.lane_dt, n_slots)) || (rc = dalloc(&ic.grp_col, (size_t)ng)) ||
        (rc = dalloc(&ic.grp_rows, (size_t)ng)) || (rc = dalloc(&ic.grp_off, (size_t)ng))) return rc;
    CU(cudaMemsetAsync(ic.lane_seg, 0xff, n_slots * 4, st));
    CU(cudaMemsetAsync(ic.lane_rows, 0, n_slots * 4, st));
    CU(cudaMemsetAsync(ic.lane_win, 0, n_slots * 2, st));
    IlAssign as{};
    as.keys = keys2; as.segs = vals2; as.elem_first = d_elem_first; as.grp_first = d_grp_first;
    as.seg_words = seg_words; as.seg_t0 = so.seg_t0; as.seg_dt = so.seg_dt; as.seg_win = so.seg_win;
    as.lane_seg = ic.lane_seg; as.lane_rows = ic.lane_rows; as.lane_series = ic.lane_series; as.grp_col = ic.grp_col; as.lane_win = ic.lane_win; as.lane_t0 = ic.lane_t0; as.lane_dt = ic.lane_dt;
    as.n_elig = (uint32_t)n_elig; as.J = J; as.cols_per_super = ic.cols_per_super;
    k_il_assign<<<(unsigned)((n_elig + 255) / 256), 256, 0, st>>>(d, as);
    k_il_group_rows<<<(unsigned)((n_slots + 255) / 256), 256, 0, st>>>(ng, ic.lane_seg, seg_words, ic.grp_rows);
    CU(cudaGetLastError());
    std::vector<uint32_t> gw(ng); std::vector<uint64_t> go(ng);
    CU(cudaMemcpyAsync(gw.data(), ic.grp_rows, (size_t)ng * 4, cudaMemcpyDeviceToHost, st));
    CU(cudaStreamSynchronize(st));
    uint64_t total = 0;
    for (uint32_t g = 0; g < ng; g++) { go[g] = total; total += (uint64_t)gw[g] * 32; }
    size_t free_b = 0, total_b = 0;
    CU(dev_mem_info(&free_b, &total_b));
    size_t headroom = (size_t)8 << 30;
    if (const char *ov = getenv("OGPU_IL_HEADROOM_MB")) headroom = (size_t)atoll(ov) << 20; /* test hook */
    if (total * 4 + headroom > free_b || dev_malloc((void **)&ic.words, total * 4) != cudaSuccess) { /* keep room for the query scratch: the general kernel serves the column */
        cudaGetLastError(); ic.words = nullptr; ic.state = -2;
        return OG_OK;
    }
    CU(cudaMemcpyAsync(ic.grp_off, go.data(), (size_t)ng * 8, cudaMemcpyHostToDevice, st));
    k_il_repack<<<(unsigned)((n_slots + 127) / 128), 128, 0, st>>>(d, col, ic.lane_seg, ic.lane_win, ic.grp_off, ic.grp_rows, ng, ic.words);
    CU(cudaGetLastError());
    timer.stop();
    CU(cudaStreamSynchronize(st));
    timer.ms(&ic.build_ms);
    ic.n_words = total; ic.n_packed = n_packed; ic.state = 1;
    return OG_OK;
}

int build_plan(og_query *q) {
    og_shard *s = q->sh;
    const QueryP &p = q->qp;
    cudaStream_t st = q->stream;
    int rc;
    Plan *pl = new Plan;
    memset((void *)pl, 0, sizeof *pl);
    q->plan = pl;
    size_t cells_dense = (size_t)q->n_groups * p.n_buckets;
    for (uint32_t c = 0; c < p.n_calls; c++) { /* dense accumulators (the result) */
        bool sel = p.calls[c].func >= OG_AGG_MIN && !(p.multi && p.calls[c].func <= OG_AGG_MAX);
        if ((rc = q->bufs.get(&q->dense[c].val, cells_dense))) return rc;
        if ((rc = q->bufs.get(&q->dense[c].ok, cells_dense))) return rc;
        if (sel && (rc = q->bufs.get(&q->dense[c].tim, cells_dense))) return rc;
    }
    /* group CSR: series sorted by (group, series) */
    std::vector<uint32_t> grp_begin(q->n_groups + 1, 0), grp_series(s->n_series);
    if (q->desc.group_mode == OG_GROUP_MAP) {
        for (uint32_t sr = 0; sr < s->n_series; sr++) grp_begin[q->series_group[sr] + 1]++;
        for (uint32_t g = 0; g < q->n_groups; g++) grp_begin[g + 1] += grp_begin[g];
        std::vector<uint32_t> cur(grp_begin.begin(), grp_begin.end() - 1);
        for (uint32_t sr = 0; sr < s->n_series; sr++) grp_series[cur[q->series_group[sr]]++] = sr;
    } else if (q->desc.group_mode == OG_GROUP_PER_SERIES) {
        for (uint32_t g = 0; g <= q->n_groups; g++) grp_begin[g] = std::min(g, s->n_series);
        std::iota(grp_series.begin(), grp_series.end(), 0u);
    } else { grp_begin[1] = s->n_series; std::iota(grp_series.begin(), grp_series.end(), 0u); }
    uint32_t *d_grp_begin, *d_grp_series;
    if ((rc = q->bufs.get(&d_grp_begin, grp_begin.size()))) return rc;
    if ((rc = q->bufs.get(&d_grp_series, grp_series.size()))) return rc;
    if ((rc = q->bufs.get(&q->d_err, 16))) return rc;
    CU(cudaMemcpyAsync(d_grp_begin, grp_begin.data(), grp_begin.size() * 4, cudaMemcpyHostToDevice, st));
    CU(cudaMemcpyAsync(d_grp_series, grp_series.data(), grp_series.size() * 4, cudaMemcpyHostToDevice, st));
    CU(cudaStreamSynchronize(st)); /* the host vectors die with this frame */
    pl->gp.grp_begin = d_grp_begin; pl->gp.grp_series = d_grp_series; pl->gp.n_groups = q->n_groups;
    for (uint32_t c = 0; c < p.n_calls; c++) pl->gp.dense[c] = q->dense[c];

    bool has_string = false;
    for (uint32_t k = 0; k < p.n_cols; k++) has_string |= p.col_type[k] == OG_TYPE_STRING;
    pl->fused = p.n_cols == 1 && p.n_filter == 0 && !has_string && !(q->desc.flags & OG_Q_NO_FUSED);
    const bool multi_ok = !pl->fused && (has_string || !(q->desc.flags & OG_Q_NO_FUSED));
    /* column-at-a-time kernel (fused_cols.cuh): const-delta time pages, <= one WHERE term, few calls per column; any number of columns */
    pl->cols = false;
    if (multi_ok && !(q->desc.flags & OG_Q_NO_FAST) && s->irregular_time_pages == 0 && s->max_seg_rows <= OG_COLS_MAXROWS &&
        (p.n_filter == 0 || (p.n_filter == 1 && p.filter[0].kind == OG_F_TERM)) && !getenv("OGPU_NO_COLS")) {
        pl->cols = true;
        for (uint32_t k = 0; k < p.n_cols; k++) {
            int n = 0;
            for (uint32_t c = 0; c < p.n_calls; c++) n += p.calls[c].col_slot == (int)k;
            if (n > OG_COLS_MAXMINE) pl->cols = false;
        }
    }
    if (has_string && !pl->cols && p.n_cols > OG_MULTI_MAXC) { set_error("a query that counts a string column may touch at most %d columns on this shard", OG_MULTI_MAXC); return OG_E_UNSUPPORTED; }
    pl->multi = pl->cols || (multi_ok && p.n_cols <= OG_MULTI_MAXC);
    q->path_used = pl->fused ? 1 : pl->cols ? 5 : pl->multi ? 4 : 0;
    const bool want_fast = pl->fused && p.col_type[0] == OG_TYPE_FLOAT && !(q->desc.flags & OG_Q_NO_FAST) && s->n_segments;
    if (want_fast && (rc = ensure_il(s, p.col_index[0], st))) return rc;
    pl->fast = want_fast && s->il[p.col_index[0]].state == 1;
    const og_shard::IlCol *ic = pl->fast ? &s->il[p.col_index[0]] : nullptr;
    pl->ic = ic;
    /* folding needs every segment index of a binning domain to cover one time range: lane groups of one rank share a column of
     * the folded matrix across segment indices (k_il_assign), and their cells must land in distinct buckets */
    pl->fold = pl->fast && ic->J != 0 && ic->aligned && q->desc.group_mode == OG_GROUP_ALL && !(q->desc.flags & OG_Q_STRICT_ORDER);

    /* chunk plan: whole series per chunk, per-series cells bounded by a memory budget */
    size_t cell_bytes_per_series = 0;
    for (uint32_t c = 0; c < p.n_calls; c++) cell_bytes_per_series += (size_t)p.n_buckets * (9 + (p.calls[c].func >= OG_AGG_MIN ? 8 : 0));
    size_t free_b = 0, total_b = 0;
    CU(dev_mem_info(&free_b, &total_b));
    size_t budget = std::min<size_t>(free_b / 3, (size_t)24 << 30);
    q->chunk_series = (uint32_t)std::max<size_t>(1, std::min<size_t>(s->n_series, budget / std::max<size_t>(1, cell_bytes_per_series)));
    if (const char *ov = getenv("OGPU_CHUNK_SERIES")) { /* test hook: force small chunks so the multi-chunk paths get exercised */
        long v = atol(ov);
        if (v > 0) q->chunk_series = (uint32_t)std::min<long>(v, (long)std::max<uint32_t>(1, s->n_series));
    }
    if (q->chunk_series < s->n_series) {
        /* lane groups are binned inside blocks of OG_IL_SUPER series: chunks that are multiples of it own whole lane groups */
        if (q->chunk_series >= OG_IL_SUPER) q->chunk_series = q->chunk_series / OG_IL_SUPER * OG_IL_SUPER;
        else q->chunk_series = std::max<uint32_t>(32, q->chunk_series & ~31u);
    }
    uint32_t max_chunk_segs = 0;
    for (uint32_t a = 0; a < s->n_series; a += q->chunk_series) {
        uint32_t b = std::min(s->n_series, a + q->chunk_series);
        max_chunk_segs = std::max(max_chunk_segs, s->h_series_seg_begin[b] - s->h_series_seg_begin[a]);
    }
    ChunkP &ch = pl->ch;
    ch.err = q->d_err; ch.flags = q->d_err + 2;
    ch.nb = p.n_buckets;
    ch.J = ic ? ic->J : 0;
    size_t chunk_cells = (size_t)std::min(q->chunk_series, s->n_series) * p.n_buckets;
    for (uint32_t c = 0; c < p.n_calls; c++) {
        bool sel = p.calls[c].func >= OG_AGG_MIN;
        if ((rc = q->bufs.get(&ch.cells[c].val, chunk_cells))) return rc;
        if ((rc = q->bufs.get(&ch.cells[c].ok, chunk_cells))) return rc;
        if (sel && (rc = q->bufs.get(&ch.cells[c].tim, chunk_cells))) return rc;
        if ((rc = q->bufs.get(&ch.edges[c].val, 2 * (size_t)max_chunk_segs))) return rc;
        if ((rc = q->bufs.get(&ch.edges[c].ok, 2 * (size_t)max_chunk_segs))) return rc;
        if (sel && (rc = q->bufs.get(&ch.edges[c].tim, 2 * (size_t)max_chunk_segs))) return rc;
    }
    if ((rc = q->bufs.get(&ch.edge_bucket, 2 * (size_t)max_chunk_segs))) return rc;
    pl->blockmerge = !pl->fold && q->desc.group_mode == OG_GROUP_ALL && !(q->desc.flags & OG_Q_STRICT_ORDER) &&
                     (s->n_series > 2 * OG_MERGE_SB || getenv("OGPU_FORCE_BLOCKMERGE") /* test hook */);
    if (pl->blockmerge) { /* block partials of the two-stage merge live in the folded cell matrix: one column per block of series */
        ch.gc_edge0 = 0; ch.gc_col0 = 0;
        ch.gc_cols = (std::min(q->chunk_series, s->n_series) + OG_MERGE_SB - 1) / OG_MERGE_SB;
        const size_t n = (size_t)p.n_buckets * ch.gc_cols;
        for (uint32_t c = 0; c < p.n_calls; c++) {
            bool sel = p.calls[c].func >= OG_AGG_MIN;
            if ((rc = q->bufs.get(&ch.gcells[c].val, n))) return rc;
            if ((rc = q->bufs.get(&ch.gcells[c].ok, n))) return rc;
            if (sel && (rc = q->bufs.get(&ch.gcells[c].tim, n))) return rc;
        }
    }
    if (pl->fold) { /* folded cell matrix: lane-group columns, their tail-window columns, then three columns per block of 32 consecutive
                       series (stitched edge windows: runs led by a head window of even / odd segment index, runs led by a tail window) */
        ch.gc_tail0 = ic->n_super * ic->cols_per_super; ch.gc_edge0 = 2 * ch.gc_tail0; ch.gc_col0 = 0;
        ch.gc_cols = ch.gc_edge0 + 3 * ((s->n_series + 31) / 32);
        const size_t n = (size_t)p.n_buckets * ch.gc_cols;
        for (uint32_t c = 0; c < p.n_calls; c++) {
            bool sel = p.calls[c].func >= OG_AGG_MIN;
            if ((rc = q->bufs.get(&ch.gcells[c].val, n))) return rc;
            if ((rc = q->bufs.get(&ch.gcells[c].ok, n))) return rc;
            if (sel && (rc = q->bufs.get(&ch.gcells[c].tim, n))) return rc;
        }
    }
    if (pl->fast) {
        pl->il.words = ic->words; pl->il.grp_off = ic->grp_off; pl->il.grp_rows = ic->grp_rows; pl->il.grp_col = ic->grp_col;
        pl->il.lane_seg = ic->lane_seg; pl->il.lane_rows = ic->lane_rows; pl->il.lane_win = ic->lane_win; pl->il.lane_series = ic->lane_series; pl->il.lane_t0 = ic->lane_t0; pl->il.lane_dt = ic->lane_dt;
        pl->fm = 0; pl->times = false;
        for (uint32_t c = 0; c < p.n_calls; c++) {
            pl->fm |= 1 << (p.calls[c].func - 1);
            if (p.calls[c].func >= OG_AGG_MIN && !(p.multi && p.calls[c].func <= OG_AGG_MAX)) pl->times = true;
        }
        pl->fm |= FM_COUNT; /* the row count also is the validity of every partial */
        q->path_used = pl->fold ? 3 : 2;
    }
    if (!pl->fused && !pl->multi) { /* generic path: materialisation tile */
        TileP &tp = pl->tp;
        tp.R = std::max<uint32_t>(1, s->max_seg_rows);
        size_t per_seg = (size_t)tp.R * (p.n_cols * 9 + 8 + 1);
        /* the decode step is one thread per page: it needs hundreds of thousands of pages in flight to hide latency, so the
         * tile is sized by free memory (a quarter of it, at most 12 GB), not by the L2 */
        size_t fb = 0, tb = 0;
        CU(dev_mem_info(&fb, &tb));
        const size_t tile_budget = std::max<size_t>((size_t)96 << 20, std::min<size_t>(fb / 4, (size_t)12 << 30));
        q->tile_segs = (uint32_t)std::max<size_t>(1, std::min<size_t>(std::max<uint32_t>(1, max_chunk_segs), tile_budget / per_seg));
        q->tile_segs = std::max<uint32_t>(32, q->tile_segs & ~31u);
        tp.S = q->tile_segs;
        for (uint32_t k = 0; k < p.n_cols; k++) {
            if ((rc = q->bufs.get(&tp.vals[k], (size_t)q->tile_segs * tp.R))) return rc;
            if ((rc = q->bufs.get(&tp.okb[k], (size_t)q->tile_segs * tp.R))) return rc;
        }
        if ((rc = q->bufs.get(&tp.times, (size_t)q->tile_segs * tp.R))) return rc;
        if ((rc = q->bufs.get(&tp.keep, (size_t)q->tile_segs * tp.R))) return rc;
    }
    q->planned = true;
    return OG_OK;
}
} // namespace
extern "C" {

OG_API int og_query_run(og_query *q) {
    if (!q) return OG_E_INVAL;
    og_shard *s = q->sh;
    CU(cudaSetDevice(s->device));
    const QueryP &p = q->qp;
    cudaStream_t st = q->stream;
    int rc;
    q->host_ready = false; q->next_group = 0; q->next_row = 0;
    if (!q->planned) {
        if (q->plan) { set_error("query plan failed earlier"); return OG_E_STATE; }
        if ((rc = build_plan(q))) return rc;
    }
    Plan *pl = (Plan *)q->plan;
    ChunkP ch = pl->ch; TileP tp = pl->tp; const GroupP &gp = pl->gp;
    size_t cells_dense = (size_t)q->n_groups * p.n_buckets;
    DirP dir = make_dir(s);
    uint32_t launches = 0, n_chunks = (s->n_series + q->chunk_series - 1) / q->chunk_series;
    while (q->main_ev.size() < 2 * (size_t)n_chunks) { cudaEvent_t e; CU(cudaEventCreate(&e)); q->main_ev.push_back(e); }
    CU(cudaMemsetAsync(q->d_err, 0, 64, st));
    CU(cudaEventRecord(q->ev0, st));
    const bool per_series = q->desc.group_mode == OG_GROUP_PER_SERIES;
    /* per-series: k_merge_per_series writes every cell of a series row; a shard without series still answers with one empty row */
    if (!per_series || s->n_series == 0) { k_init_dense<<<(unsigned)((cells_dense + 255) / 256), 256, 0, st>>>(p, gp); launches++; }
    /* folded runs touch the per-series cells only on fallback paths: their validity bytes are cleared only after a run that used them */
    const bool clear_cells = !pl->fold || q->cells_dirty || n_chunks > 1;
    uint64_t segs_scanned = 0; uint32_t ci = 0, chunks_run = 0;
    for (uint32_t a = 0; a < s->n_series; a += q->chunk_series, ci++) {
        if (q->aborted) { cudaStreamSynchronize(st); set_error("query aborted"); return OG_E_ABORTED; }
        uint32_t b = std::min(s->n_series, a + q->chunk_series);
        ch.series_begin = a; ch.series_end = b;
        ch.seg_begin = s->h_series_seg_begin[a]; ch.seg_end = s->h_series_seg_begin[b];
        uint32_t nseg = ch.seg_end - ch.seg_begin;
        const size_t chunk_cells = (size_t)(b - a) * p.n_buckets;
        if (nseg == 0) {
            if (per_series) { /* series without segments still own dense rows: write them as empty */
                for (uint32_t c = 0; c < p.n_calls; c++) CU(cudaMemsetAsync(ch.cells[c].ok, 0, chunk_cells, st));
                k_merge_per_series<<<dim3((unsigned)((chunk_cells + 255) / 256), p.n_calls), 256, 0, st>>>(p, ch, gp);
                launches++;
            }
            continue;
        }
        segs_scanned += nseg;
        if (clear_cells) for (uint32_t c = 0; c < p.n_calls; c++) CU(cudaMemsetAsync(ch.cells[c].ok, 0, chunk_cells, st));
        /* folded cells are per chunk: a lane group that straddles chunks contributes to its column once per chunk */
        if (pl->fold || pl->blockmerge) for (uint32_t c = 0; c < p.n_calls; c++) CU(cudaMemsetAsync(ch.gcells[c].ok, 0, (size_t)p.n_buckets * ch.gc_cols, st));
        if (pl->fold && ci > 0) CU(cudaMemsetAsync(ch.flags + 1, 0, sizeof(int), st)); /* "edge windows written" is per chunk (the run's first chunk starts from the cleared error buffer) */
        CU(cudaEventRecord(q->main_ev[2 * chunks_run], st));
        if (pl->fused) {
            const uint32_t *gl = nullptr; uint32_t gn = nseg;
            if (pl->fast) {
                const og_shard::IlCol &ic = *pl->ic;
                /* lane groups of this chunk: those of the blocks of OG_IL_SUPER series it touches (a group that straddles the chunk
                 * boundary runs in both chunks, with the lanes of each) */
                uint32_t g0 = 0, g1 = ic.n_groups;
                if (ic.J) { g0 = ic.super_grp_first[a / OG_IL_SUPER]; g1 = ic.super_grp_first[std::min<uint32_t>(ic.n_super, (b + OG_IL_SUPER - 1) / OG_IL_SUPER)]; }
                launch_fast(pl->fm, pl->times, pl->fold, pl->il, g0, g1, p, ch, st); launches++;
                /* leftovers of this chunk: a contiguous range of the sorted list */
                auto lo = std::lower_bound(ic.gen_host.begin(), ic.gen_host.end(), ch.seg_begin);
                auto hi = std::lower_bound(ic.gen_host.begin(), ic.gen_host.end(), ch.seg_end);
                gl = ic.gen_list + (lo - ic.gen_host.begin()); gn = (uint32_t)(hi - lo);
            }
            if (gn) {
                switch (p.n_calls) {
                case 1: launch_fused<1>(dir, p, ch, gl, gn, st); break;
                case 2: launch_fused<2>(dir, p, ch, gl, gn, st); break;
                case 3: launch_fused<3>(dir, p, ch, gl, gn, st); break;
                case 4: launch_fused<4>(dir, p, ch, gl, gn, st); break;
                case 5: launch_fused<5>(dir, p, ch, gl, gn, st); break;
                case 6: launch_fused<6>(dir, p, ch, gl, gn, st); break;
                case 7: launch_fused<7>(dir, p, ch, gl, gn, st); break;
                default: launch_fused<8>(dir, p, ch, gl, gn, st); break;
                }
                launches++;
            }
        } else if (pl->cols) {
            launch_cols(p, dir, ch, nseg, st);
        } else if (pl->multi) {
            launch_multi(p, dir, ch, nseg, st);
            launches++;
        } else {
            for (uint32_t t0 = ch.seg_begin; t0 < ch.seg_end; t0 += q->tile_segs) {
                tp.tile_begin = t0; tp.tile_end = std::min(ch.seg_end, t0 + q->tile_segs);
                uint32_t n = tp.tile_end - tp.tile_begin;
                dim3 g((n + 127) / 128, p.n_cols + 1);
                k_decode_tile<<<g, 128, 0, st>>>(dir, p, tp, q->d_err);
                size_t rows_total = (size_t)tp.S * tp.R;
                k_filter_tile<<<(unsigned)((rows_total + 255) / 256), 256, 0, st>>>(dir, p, tp);
                k_window_reduce<<<(n + 127) / 128, 128, 0, st>>>(dir, p, tp, ch);
                launches += 3;
            }
        }
        CU(cudaEventRecord(q->main_ev[2 * chunks_run + 1], st));
        chunks_run++;
        if (pl->fold) k_fix_edges_fold<<<(unsigned)(((size_t)((b - a + 31) / 32) * ch.J * 32 + 127) / 128), 128, 0, st>>>(dir, p, ch);
        else k_fix_edges<<<(nseg + 127) / 128, 128, 0, st>>>(dir, p, ch);
        if (per_series) k_merge_per_series<<<dim3((unsigned)((chunk_cells + 255) / 256), p.n_calls), 256, 0, st>>>(p, ch, gp);
        else if (pl->blockmerge) k_merge_all_blocks<<<dim3((p.n_buckets + 127) / 128, (b - a + OG_MERGE_SB - 1) / OG_MERGE_SB, p.n_calls), 128, 0, st>>>(p, ch, gp);
        else k_merge_groups<<<dim3((unsigned)((cells_dense + 127) / 128), p.n_calls), 128, 0, st>>>(p, ch, gp); /* returns at once when no per-series cell was written */
        launches += 2;
        if (pl->fold || pl->blockmerge) { k_merge_folded<<<dim3((unsigned)(((size_t)p.n_buckets * 32 + 127) / 128), p.n_calls), 128, 0, st>>>(p, ch, gp); launches++; }
    }
    CU(cudaEventRecord(q->ev1, st));
    CU(cudaGetLastError());
    CU(cudaStreamSynchronize(st));
    int err[16];
    CU(cudaMemcpy(err, q->d_err, 64, cudaMemcpyDeviceToHost));
    if (getenv("OGPU_IL_STATS")) {
        /* warp cycles waiting for ring batches / over the warp's lifetime / before the first round / after the last round (OG_IL_STATS builds) */
        unsigned long long wait, life, pro, epi;
        memcpy(&wait, err + 8, 8); memcpy(&life, err + 10, 8); memcpy(&pro, err + 12, 8); memcpy(&epi, err + 14, 8);
        const double pc = life ? 100.0 / (double)life : 0.0;
        fprintf(stderr, "[ogpu] fused rounds: common %d rare %d (lanes not resident in %d, sit-outs %d); warp cycles: %llu waiting for batches of %llu (%.1f %%), "
                "prologue %llu (%.1f %%), epilogue %llu (%.1f %%)\n",
                err[4], err[5], err[6], err[7], wait, life, pc * (double)wait, pro, pc * (double)pro, epi, pc * (double)epi);
    }
    q->cells_dirty = err[2] != 0;
    if (err[0]) { set_error("segment %d failed to decode (device code %d)", err[1], err[0]); return map_dev_err(err[0]); }
    float ms = 0; cudaEventElapsedTime(&ms, q->ev0, q->ev1);
    double main_ms = 0;
    for (uint32_t i = 0; i < chunks_run; i++) { float m = 0; cudaEventElapsedTime(&m, q->main_ev[2 * i], q->main_ev[2 * i + 1]); main_ms += m; }
    og_stats &stt = q->stats;
    uint64_t keep_pb = stt.page_bytes, keep_rows = stt.rows_decoded, keep_segs = stt.segments_scanned; /* directory sums do not change between runs */
    memset(&stt, 0, sizeof stt);
    stt.kernel_ms = ms; stt.main_kernel_ms = main_ms; stt.kernel_launches = launches; stt.path = q->path_used;
    stt.page_bytes = keep_pb; stt.rows_decoded = keep_pb ? keep_rows : s->n_rows; stt.segments_scanned = keep_pb ? keep_segs : segs_scanned;
    stt.dir_bytes = (uint64_t)segs_scanned * 32; /* SURVEY §8d accounting: 32 B of directory per scanned segment */
    stt.out_bytes = 0;
    for (uint32_t c = 0; c < p.n_calls; c++) stt.out_bytes += cells_dense * (9 + (q->dense[c].tim ? 8 : 0));
    if (p.n_cols == 1 && p.col_type[0] == OG_TYPE_FLOAT) {
        /* a query of another thread may be building this copy (ensure_il marks it -1 until it is ready): read it under the
           build's lock, so a query never reports a half-built copy as "no eligible page" */
        std::lock_guard<std::mutex> il_lock(s->il_mu);
        if (p.col_index[0] < (int)s->il.size()) {
            const og_shard::IlCol &ic = s->il[p.col_index[0]];
            stt.il_state = ic.state; stt.il_build_ms = ic.build_ms; stt.il_bytes = ic.n_words * 4; stt.il_packed_segments = ic.state == 1 ? ic.n_packed : 0;
            stt.general_segments = ic.state == 1 ? (uint64_t)ic.gen_host.size() : s->n_segments;
        }
    }
    stt.per_series_cells_used = err[2] != 0;
    q->ran = true;
    return OG_OK;
}

OG_API int og_query_dense(og_query *q, og_dense_view *out) {
    if (!q || !out) return OG_E_INVAL;
    if (!q->ran) { set_error("og_query_dense before og_query_run"); return OG_E_STATE; }
    const QueryP &p = q->qp;
    /* without GROUP BY time() the single interval row carries time 0 (BuildEmptyIntervalRec !hasInterval, record.go:1328-1331) */
    out->n_groups = q->n_groups; out->n_buckets = p.n_buckets; out->start = q->desc.interval ? p.start : 0; out->interval = q->desc.interval ? p.interval : 0;
    out->n_cols = p.n_calls;
    for (uint32_t c = 0; c < p.n_calls; c++) {
        q->dense_cols[c].values = q->dense[c].val; q->dense_cols[c].valid = q->dense[c].ok; q->dense_cols[c].times = q->dense[c].tim;
        q->dense_cols[c].type = p.calls[c].out_type; q->dense_cols[c].func = p.calls[c].func;
    }
    out->cols = q->dense_cols; out->stream = q->stream;
    return OG_OK;
}

} /* extern "C" */
namespace {
__global__ void k_sum_page_bytes(DirP d, QueryP q, int64_t tmin, int64_t tmax, unsigned long long *out /*[0] bytes [1] rows [2] segs*/) {
    uint32_t seg = blockIdx.x * blockDim.x + threadIdx.x;
    if (seg >= d.n_segments) return;
    if (d.seg_tmax[seg] < tmin || d.seg_tmin[seg] > tmax) return;
    unsigned long long b = d.page_len[(size_t)d.n_columns * d.n_segments + seg];
    for (uint32_t k = 0; k < q.n_cols; k++) b += d.page_len[(size_t)q.col_index[k] * d.n_segments + seg];
    atomicAdd(&out[0], b); atomicAdd(&out[1], (unsigned long long)d.seg_rows[seg]); atomicAdd(&out[2], 1ull);
}
} // namespace
extern "C" {

OG_API int og_query_stats(const og_query *q, og_stats *out) {
    if (!q || !out) return OG_E_INVAL;
    og_query *mq = const_cast<og_query *>(q);
    if (q->ran && q->stats.page_bytes == 0) {
        CU(cudaSetDevice(q->sh->device));
        Scratch tmp;
        unsigned long long *d_o; int rc = tmp.get(&d_o, 3); if (rc) return rc;
        cudaMemset(d_o, 0, 24);
        if (q->sh->n_segments) k_sum_page_bytes<<<(q->sh->n_segments + 255) / 256, 256>>>(make_dir(q->sh), q->qp, q->qp.tmin, q->qp.tmax, d_o);
        unsigned long long h[3]; CU(cudaMemcpy(h, d_o, 24, cudaMemcpyDeviceToHost));
        mq->stats.page_bytes = h[0]; mq->stats.rows_decoded = h[1]; mq->stats.segments_scanned = h[2];
    }
    *out = q->stats;
    return OG_OK;
}

OG_API int og_query_merge_dense(og_query *q, const og_dense_view *other) {
    if (!q || !other) return OG_E_INVAL;
    if (!q->ran) return OG_E_STATE;
    const QueryP &p = q->qp;
    if (other->n_groups != q->n_groups || other->n_buckets != p.n_buckets || other->n_cols != p.n_calls) { set_error("dense shapes differ"); return OG_E_INVAL; }
    if (other->start != (q->desc.interval ? p.start : 0) || other->interval != (q->desc.interval ? p.interval : 0)) {
        set_error("dense grids differ (start %lld vs %lld, interval %lld vs %lld): create the queries with OG_Q_QUERY_GRID", (long long)other->start,
                  (long long)(q->desc.interval ? p.start : 0), (long long)other->interval, (long long)(q->desc.interval ? p.interval : 0));
        return OG_E_INVAL;
    }
    CU(cudaSetDevice(q->sh->device));
    GroupP mine, oth; memset(&mine, 0, sizeof mine); memset(&oth, 0, sizeof oth);
    mine.n_groups = oth.n_groups = q->n_groups;
    for (uint32_t c = 0; c < p.n_calls; c++) {
        /* the cells are raw bits: a record of other calls or types would be read as this one's (a count as a sum, int bits as doubles) */
        if (other->cols[c].func != p.calls[c].func || other->cols[c].type != p.calls[c].out_type) {
            set_error("dense column %u: func %d type %d, this query's is func %d type %d", c, other->cols[c].func, other->cols[c].type, p.calls[c].func,
                      p.calls[c].out_type);
            return OG_E_INVAL;
        }
        mine.dense[c] = q->dense[c];
        oth.dense[c].val = (uint64_t *)other->cols[c].values; oth.dense[c].ok = other->cols[c].valid; oth.dense[c].tim = other->cols[c].times;
        if ((q->dense[c].tim != nullptr) != (oth.dense[c].tim != nullptr)) { set_error("dense column %u: times presence differs", c); return OG_E_INVAL; }
    }
    size_t total = (size_t)q->n_groups * p.n_buckets;
    k_merge_dense<<<(unsigned)((total + 255) / 256), 256, 0, q->stream>>>(p, mine, oth);
    CU(cudaGetLastError());
    CU(cudaStreamSynchronize(q->stream));
    q->host_ready = false;
    return OG_OK;
}

/* KeyCursor.Next: TransIntervalRec2Rec (lib/record/record.go:1340-1358) in slices of ChunkSizeNum (agg_tagset_cursor.go:993-1006) */
OG_API int og_query_next(og_query *q, og_record_view *out) {
    if (!q || !out) return OG_E_INVAL;
    if (!q->ran) { set_error("og_query_next before og_query_run"); return OG_E_STATE; }
    if (q->aborted) return OG_E_ABORTED;
    const QueryP &p = q->qp;
    size_t total = (size_t)q->n_groups * p.n_buckets;
    if (!q->host_ready) {
        CU(cudaSetDevice(q->sh->device));
        for (uint32_t c = 0; c < p.n_calls; c++) {
            q->h_val[c].resize(total); q->h_ok[c].resize(total);
            CU(cudaMemcpy(q->h_val[c].data(), q->dense[c].val, total * 8, cudaMemcpyDeviceToHost));
            CU(cudaMemcpy(q->h_ok[c].data(), q->dense[c].ok, total, cudaMemcpyDeviceToHost));
            if (q->dense[c].tim) { q->h_tim[c].resize(total); CU(cudaMemcpy(q->h_tim[c].data(), q->dense[c].tim, total * 8, cudaMemcpyDeviceToHost)); }
        }
        q->host_ready = true; q->next_group = 0; q->next_row = 0;
    }
    int chunk = q->desc.chunk_size > 0 ? q->desc.chunk_size : 1024;
    uint32_t nc = p.n_calls;
    q->rv_val.assign(nc, {}); q->rv_bitmap.assign(nc, {}); q->rv_coltimes.assign(nc, {}); q->rv_times.clear(); q->rv_cols.assign(nc, og_colval_view{});
    while (q->next_group < q->n_groups) {
        uint32_t g = q->next_group;
        std::vector<int32_t> nil(nc, 0);
        int rows = 0;
        uint32_t b = q->next_row;
        /* a slice covers `chunk` interval rows; empty rows inside it are dropped */
        uint32_t b_end = (uint32_t)std::min<uint64_t>(p.n_buckets, (uint64_t)b + (uint64_t)chunk);
        for (; b < b_end; b++) {
            const uint32_t bb = q->desc.ascending ? b : p.n_buckets - 1 - b; /* descending: latest window first */
            size_t i = (size_t)g * p.n_buckets + bb;
            bool any = false;
            for (uint32_t c = 0; c < nc; c++) any |= q->h_ok[c][i] != 0;
            if (!any) continue;
            int64_t row_time = p.start + (int64_t)bb * p.interval;
            if (q->desc.interval == 0) row_time = 0;
            for (uint32_t c = 0; c < nc; c++) {
                bool ok = q->h_ok[c][i] != 0;
                if ((size_t)(rows >> 3) >= q->rv_bitmap[c].size()) q->rv_bitmap[c].push_back(0);
                if (ok) {
                    q->rv_bitmap[c][rows >> 3] |= (uint8_t)(1 << (rows & 7));
                    if (p.calls[c].out_type == OG_TYPE_BOOL) q->rv_val[c].push_back((uint8_t)(q->h_val[c][i] != 0));
                    else { const uint8_t *pv = (const uint8_t *)&q->h_val[c][i]; q->rv_val[c].insert(q->rv_val[c].end(), pv, pv + 8); }
                } else nil[c]++;
                if (q->dense[c].tim) {
                    if (p.multi) q->rv_coltimes[c].push_back(ok ? q->h_tim[c][i] : 0);
                    else if (ok) row_time = q->h_tim[c][i]; /* single-call selector: the row carries the point's time */
                }
            }
            q->rv_times.push_back(row_time);
            rows++;
        }
        q->next_row = b_end;
        if (q->next_row >= p.n_buckets) { q->next_group++; q->next_row = 0; }
        if (rows == 0) continue;
        for (uint32_t c = 0; c < nc; c++) {
            og_colval_view &v = q->rv_cols[c];
            v.val = q->rv_val[c].data(); v.val_bytes = q->rv_val[c].size(); v.bitmap = q->rv_bitmap[c].data();
            v.times = (p.multi && q->dense[c].tim) ? q->rv_coltimes[c].data() : nullptr;
            v.type = p.calls[c].out_type; v.len = rows; v.nil_count = nil[c]; v.bitmap_offset = 0;
        }
        out->n_cols = nc; out->cols = q->rv_cols.data(); out->times = q->rv_times.data(); out->rows = rows; out->group = g;
        out->sid = q->desc.group_mode == OG_GROUP_PER_SERIES ? q->sh->sids[g] : 0;
        return OG_OK;
    }
    return OG_EOF;
}

/* =============================================== materialise path =============================================== */
} /* extern "C" */
namespace {
/* decode [seg_begin, seg_end) of one column into dense non-null values (ColVal.Val layout, reader.go:504-579) */
__global__ void k_decode_column(DirP d, uint32_t column, int type, uint32_t seg_begin, uint32_t seg_end, uint8_t *out, uint64_t stride,
                                uint32_t *rows_out, uint8_t *bitmap_out, uint32_t bitmap_stride, int *err) {
    uint32_t seg = seg_begin + blockIdx.x * blockDim.x + threadIdx.x;
    if (seg >= seg_end) return;
    uint8_t *o = out + (size_t)(seg - seg_begin) * stride;
    uint32_t rows = d.seg_rows[seg];
    size_t pi = (size_t)column * d.n_segments + seg;
    if (column == d.n_columns) { /* time column */
        TimeDesc t;
        int rc = parse_time_page(d.data + d.page_off[pi], d.page_len[pi], t);
        if (rc == D_OK) {
            TimeIter it; it.init(t);
            for (uint32_t i = 0; i < t.rows; i++) ((int64_t *)o)[i] = it.next();
            it.finish(); rc = it.err;
        }
        if (rc != D_OK) report_err(err, rc, seg);
        if (rows_out) rows_out[seg - seg_begin] = rows;
        return;
    }
    uint32_t len = d.page_len[pi];
    uint8_t *bm = bitmap_out ? bitmap_out + (size_t)(seg - seg_begin) * bitmap_stride : nullptr;
    if (len == 0) {
        if (rows_out) rows_out[seg - seg_begin] = 0;
        if (bm) for (uint32_t i = 0; i < (rows + 7) / 8; i++) bm[i] = 0;
        return;
    }
    ColIter it;
    it.init(d.data + d.page_off[pi], len, type, rows);
    int rc = it.err;
    if (rc == D_OK && type == OG_TYPE_STRING) rc = D_UNSUPPORTED; /* string values are never decoded on the device */
    if (rc == D_OK) {
        const PageHdr &h = it.h;
        for (uint32_t r = 0, j = 0; r < rows; r++) {
            uint64_t v;
            if (!it.next(v)) continue;
            if (type == OG_TYPE_BOOL) o[j++] = (uint8_t)v; else ((uint64_t *)o)[j++] = v;
        }
        it.finish(); rc = it.err;
        if (rows_out) rows_out[seg - seg_begin] = h.rows - h.nil_count;
        if (bm) { /* AppendBitmap re-packed at offset 0 (lib/record/column.go:79-112) */
            for (uint32_t i = 0; i < (rows + 7) / 8; i++) {
                uint8_t v = 0;
                for (uint32_t k = 0; k < 8 && i * 8 + k < rows; k++) v |= (uint8_t)(hdr_row_valid(h, i * 8 + k) ? 1 : 0) << k;
                bm[i] = v;
            }
        }
    }
    if (rc != D_OK) report_err(err, rc, seg);
}
} // namespace
extern "C" {

OG_API int og_decode_column_device(og_shard *s, uint32_t column, uint32_t seg_begin, uint32_t seg_end, void *d_values,
                                   uint64_t value_stride_bytes, uint32_t *d_rows_out) {
    if (!s || !d_values || column > s->n_columns || seg_begin > seg_end || seg_end > s->n_segments) { set_error("bad argument"); return OG_E_INVAL; }
    CU(cudaSetDevice(s->device));
    if (seg_begin == seg_end) return OG_OK;
    int *d_err; int rc = dalloc(&d_err, 2); if (rc) return rc;
    cudaMemset(d_err, 0, 8);
    int type = column == s->n_columns ? OG_TYPE_INT : s->col_types[column];
    uint32_t n = seg_end - seg_begin;
    k_decode_column<<<(n + 127) / 128, 128>>>(make_dir(s), column, type, seg_begin, seg_end, (uint8_t *)d_values, value_stride_bytes, d_rows_out, nullptr, 0, d_err);
    int err[2]; cudaError_t e = cudaMemcpy(err, d_err, 8, cudaMemcpyDeviceToHost); dev_free(d_err);
    if (e != cudaSuccess) return cuda_fail(e, "k_decode_column", __FILE__, __LINE__);
    if (err[0]) { set_error("segment %d failed to decode (device code %d)", err[1], err[0]); return map_dev_err(err[0]); }
    return OG_OK;
}

/* one segment -> Record view in pinned host memory (the KeyCursor.Next of a non-aggregating reader) */
/* descending scans hand every segment over reversed: values, validity bits and times (reader.go:516-519,1035-1042 reverseXxxValues) */
__global__ void k_reverse_segment(uint8_t *vals, uint32_t elem_bytes, uint32_t n_vals, uint8_t *bitmap, uint32_t rows) {
    for (uint32_t i = threadIdx.x; i < n_vals / 2; i += blockDim.x) {
        const uint32_t j = n_vals - 1 - i;
        if (elem_bytes == 8) { uint64_t *v = (uint64_t *)vals; const uint64_t a = v[i]; v[i] = v[j]; v[j] = a; }
        else { const uint8_t a = vals[i]; vals[i] = vals[j]; vals[j] = a; }
    }
    if (!bitmap) return;
    __syncthreads();
    __shared__ uint8_t sbm[8192]; /* rows <= 65536 */
    const uint32_t nb = (rows + 7) / 8;
    for (uint32_t i = threadIdx.x; i < nb; i += blockDim.x) sbm[i] = bitmap[i];
    __syncthreads();
    for (uint32_t i = threadIdx.x; i < nb; i += blockDim.x) {
        uint8_t o = 0;
        for (uint32_t k = 0; k < 8 && i * 8 + k < rows; k++) { const uint32_t src = rows - 1 - (i * 8 + k); o |= (uint8_t)((sbm[src >> 3] >> (src & 7)) & 1) << k; }
        bitmap[i] = o;
    }
}
} // extern "C"
static int decode_segment_impl(og_shard *s, uint32_t segment, uint32_t flags, og_record_view *out);
extern "C" {
OG_API int og_decode_segment(og_shard *s, uint32_t segment, og_record_view *out) { return decode_segment_impl(s, segment, 0, out); }
OG_API int og_decode_segment_ex(og_shard *s, uint32_t segment, uint32_t flags, og_record_view *out) { return decode_segment_impl(s, segment, flags, out); }
} // extern "C"
static int decode_segment_impl(og_shard *s, uint32_t segment, uint32_t flags, og_record_view *out) {
    if (!s || !out || segment >= s->n_segments) { set_error("bad argument"); return OG_E_INVAL; }
    CU(cudaSetDevice(s->device));
    uint32_t R = std::max<uint32_t>(1, s->max_seg_rows);
    size_t ncol1 = (size_t)s->n_columns + 1;
    size_t val_stride = (size_t)R * 8, bm_stride = (((size_t)R + 7) / 8 + 7) & ~(size_t)7;
    size_t need = ncol1 * (val_stride + bm_stride + 16);
    if (s->d_seg_buf_bytes < need || s->h_seg_buf_bytes < need) { /* a failed allocation leaves a buffer null with size 0 */
        dev_free(s->d_seg_buf); s->d_seg_buf = nullptr; s->d_seg_buf_bytes = 0;
        if (s->h_seg_buf) cudaFreeHost(s->h_seg_buf);
        s->h_seg_buf = nullptr; s->h_seg_buf_bytes = 0;
        CU(dev_malloc(&s->d_seg_buf, need)); s->d_seg_buf_bytes = need;
        CU(cudaMallocHost(&s->h_seg_buf, need)); s->h_seg_buf_bytes = need;
    }
    uint8_t *dv = (uint8_t *)s->d_seg_buf, *dbm = dv + ncol1 * val_stride;
    uint32_t *drows = (uint32_t *)(dbm + ncol1 * bm_stride);
    int *d_err; int rc = dalloc(&d_err, 2); if (rc) return rc;
    cudaMemset(d_err, 0, 8);
    DirP dir = make_dir(s);
    for (uint32_t c = 0; c <= s->n_columns; c++) {
        int type = c == s->n_columns ? OG_TYPE_INT : s->col_types[c];
        k_decode_column<<<1, 32>>>(dir, c, type, segment, segment + 1, dv + c * val_stride, val_stride, drows + c, dbm + c * bm_stride, (uint32_t)bm_stride, d_err);
    }
    int err[2]; cudaError_t e = cudaMemcpy(err, d_err, 8, cudaMemcpyDeviceToHost); dev_free(d_err);
    if (e != cudaSuccess) return cuda_fail(e, "k_decode_column", __FILE__, __LINE__);
    if (err[0]) { set_error("segment %d failed to decode (device code %d)", err[1], err[0]); return map_dev_err(err[0]); }
    if (flags & OG_DECODE_DESCENDING) {
        if (R > 65536) { set_error("descending materialisation supports segments of up to 65536 rows"); return OG_E_UNSUPPORTED; }
        uint32_t hr[65]; /* non-null counts per column, rows in the last slot */
        CU(cudaMemcpy(hr, drows, (ncol1) * 4, cudaMemcpyDeviceToHost));
        const uint32_t rows_seg = hr[s->n_columns];
        for (uint32_t c = 0; c <= s->n_columns; c++) {
            const bool is_time = c == s->n_columns;
            const uint32_t eb = (!is_time && s->col_types[c] == OG_TYPE_BOOL) ? 1 : 8;
            k_reverse_segment<<<1, 256>>>(dv + c * val_stride, eb, is_time ? rows_seg : hr[c], is_time ? nullptr : dbm + c * bm_stride, rows_seg);
        }
        CU(cudaGetLastError());
    }
    CU(cudaMemcpy(s->h_seg_buf, s->d_seg_buf, need, cudaMemcpyDeviceToHost));
    uint8_t *hv = (uint8_t *)s->h_seg_buf, *hbm = hv + ncol1 * val_stride;
    uint32_t *hrows = (uint32_t *)(hbm + ncol1 * bm_stride);
    uint32_t rows = hrows[s->n_columns];
    s->seg_views.assign(s->n_columns, og_colval_view{});
    for (uint32_t c = 0; c < s->n_columns; c++) {
        og_colval_view &v = s->seg_views[c];
        uint32_t nv = hrows[c];
        v.val = hv + c * val_stride; v.val_bytes = (uint64_t)nv * (s->col_types[c] == OG_TYPE_BOOL ? 1 : 8);
        v.bitmap = hbm + c * bm_stride; v.times = nullptr; v.type = s->col_types[c]; v.len = (int32_t)rows; v.nil_count = (int32_t)(rows - nv); v.bitmap_offset = 0;
    }
    out->n_cols = s->n_columns; out->cols = s->seg_views.data(); out->times = (const int64_t *)(hv + s->n_columns * val_stride); out->rows = (int32_t)rows; out->group = 0;
    /* series id of the segment */
    uint32_t sr = (uint32_t)(std::upper_bound(s->h_series_seg_begin.begin(), s->h_series_seg_begin.end(), segment) - s->h_series_seg_begin.begin()) - 1;
    out->sid = s->sids[sr];
    return OG_OK;
}
