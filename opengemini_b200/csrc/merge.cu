/*
 * merge.cu — og_shard_open_files: the ordered and out-of-order files of one shard opened as ONE og_shard.
 *
 * The reference merges a shard's files for every series of every query (include/ogpu.h lists the code).  Here the merge runs
 * once, when the shard is opened:
 *
 *   host   check every description (check_desc), union of columns by name and of series by sid, the ordered segments of a
 *          series in file order (overlapping ordered files are refused), one H2D per file into one data buffer with rebased
 *          page offsets; the whole file set is validated and its Snappy pages transcoded by shard_finalize, so the merge only
 *          sees codecs ColIter / TimeIter decode.
 *   order  the rows of one time are ranked oldest first: ordered files, then out-of-order files, each in file sequence.
 *   span   per series with out-of-order rows: the hull [min, max] of its out-of-order segments' time ranges, widened to the
 *          ordered segments it overlaps.  Those ordered segments and every out-of-order segment of the series are rewritten;
 *          every other segment keeps its bytes and its directory entry.
 *   device per batch of spans (scratch ~ rows in the batch, under a device-memory budget):
 *          k_merge_decode   one thread per source segment: rows of every union column, laid out span by span, sources of a span
 *                           in file-sequence order
 *          StableSortPairs  by time inside each span (cub segmented sort): rows of equal time stay in file order, oldest first
 *          k_merge_heads    first row of each run of equal times; a time repeated inside one file is OG_E_CORRUPT
 *          k_merge_combine  one thread per run: each column takes its newest non-null value (mergeRecRow, record.go:468-505),
 *                           written into 1000-row segment slots (lib/util/util.go:72)
 *          encode_pages     the adaptive encoders of og_encode_pages (encode.cu), raw page for a float segment Gorilla refuses
 *   finish the new pages are appended behind the data, the directory is rebuilt, and shard_finalize validates the result.
 */
#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <map>
#include <string>
#include <vector>

#include <cub/device/device_scan.cuh>
#include <cub/device/device_segmented_sort.cuh>

#include "decode.cuh"
#include "internal.h"

namespace ogpu {

int shard_finalize(og_shard *s, bool scan_snappy); /* api.cu */
int check_desc(const og_shard_desc *d);            /* api.cu */
int upload_dir(og_shard *s, const uint32_t *series_seg_begin, const int64_t *seg_tmin, const int64_t *seg_tmax, const uint64_t *page_off,
               const uint32_t *page_len, const uint64_t *sids); /* api.cu */
int encode_pages(int32_t type, int32_t is_time, const void *d_values, const uint8_t *d_valid, const uint32_t *d_rows, uint32_t n_segments,
                 uint32_t rps, uint8_t *d_out, uint64_t out_cap, uint64_t *d_page_off, uint32_t *d_page_len, uint64_t *total_bytes_out,
                 bool nan_raw); /* encode.cu */

#define MERGE_RPS 1000u           /* rows per rewritten segment: lib/util/util.go:72 */
#define MERGE_PAGE_BOUND 8704u    /* largest page the encoders write for 1000 rows (encode.cu PAGE_STRIDE) */

/* the part of the device directory the merge reads */
struct SrcDir {
    const uint8_t *data; const uint64_t *page_off; const uint32_t *page_len; const uint32_t *seg_rows;
    uint32_t n_segments, n_columns;
};

enum { M_STRING = 100, M_REPEAT = 101 };
struct MergeErr { int code, seg, col, span, file; long long time; };

__device__ __forceinline__ bool merge_claim(MergeErr *e, int code) { return atomicCAS(&e->code, 0, code) == 0; }

/* one thread per source segment of the batch: decode its rows into the batch's row arrays */
__global__ void k_merge_decode(SrcDir d, const int32_t *col_types, uint32_t n, const uint32_t *src_seg, const uint32_t *src_row0,
                               const uint32_t *src_file, const uint32_t *src_span, uint32_t R, int64_t *times, uint32_t *row_file,
                               uint32_t *row_span, uint64_t *cells, uint8_t *ok, MergeErr *err) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint32_t seg = src_seg[i], r0 = src_row0[i], rows = d.seg_rows[seg];
    const size_t ti = (size_t)d.n_columns * d.n_segments + seg;
    TimeDesc t;
    int rc = parse_time_page(d.data + d.page_off[ti], d.page_len[ti], t);
    if (rc == D_OK && t.rows != rows) rc = D_CORRUPT;
    if (rc == D_OK) {
        TimeIter it; it.init(t);
        for (uint32_t k = 0; k < rows; k++) { times[r0 + k] = it.next(); row_file[r0 + k] = src_file[i]; row_span[r0 + k] = src_span[i]; }
        it.finish(); rc = it.err;
    }
    if (rc != D_OK) { if (merge_claim(err, rc)) err->seg = (int)seg; return; }
    for (uint32_t c = 0; c < d.n_columns; c++) {
        const size_t pi = (size_t)c * d.n_segments + seg;
        uint64_t *cv = cells + (size_t)c * R + r0;
        uint8_t *ov = ok + (size_t)c * R + r0;
        ColIter ci;
        ci.init(d.data + d.page_off[pi], d.page_len[pi], col_types[c], rows);
        if (ci.err == D_OK && ci.kind == ColIter::K_NULLMAP) { /* a string value: there is no device string encoder */
            if (merge_claim(err, M_STRING)) { err->seg = (int)seg; err->col = (int)c; err->span = (int)src_span[i]; }
            return;
        }
        for (uint32_t k = 0; k < rows; k++) {
            uint64_t v = 0;
            const bool has = ci.next(v);
            cv[k] = has ? v : 0; ov[k] = has ? 1 : 0;
        }
        ci.finish();
        if (ci.err != D_OK) { if (merge_claim(err, ci.err)) err->seg = (int)seg; return; }
    }
}

__global__ void k_merge_iota(uint32_t *v, uint32_t n) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) v[i] = i;
}

/* head[i] = 1 where sorted row i starts a run of equal times in its span; head[R] = 0 so the exclusive scan ends in the total */
__global__ void k_merge_heads(const int64_t *t, const uint32_t *perm, const uint32_t *row_file, const uint32_t *row_span, uint32_t R,
                              uint32_t *head, MergeErr *err) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i > R) return;
    if (i == R) { head[i] = 0; return; }
    const bool h = i == 0 || row_span[i] != row_span[i - 1] || t[i] != t[i - 1];
    head[i] = h ? 1u : 0u;
    if (!h && row_file[perm[i]] == row_file[perm[i - 1]] && merge_claim(err, M_REPEAT)) {
        err->span = (int)row_span[i]; err->file = (int)row_file[perm[i]]; err->time = (long long)t[i];
    }
}

/* out_begin[s] = output row of span s's first row (s = n_spans: the batch's total) */
__global__ void k_merge_span_out(const uint32_t *span_row0, uint32_t n_spans, const uint32_t *oidx, uint32_t *out_begin) {
    const uint32_t s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s <= n_spans) out_begin[s] = oidx[span_row0[s]];
}

/* one thread per run of equal times: the row rule, then the merged row into its 1000-row segment slot */
__global__ void k_merge_combine(const int64_t *t, const uint32_t *perm, const uint32_t *row_span, const uint32_t *head,
                                const uint32_t *oidx, const uint32_t *out_begin, const uint32_t *seg_base, const int32_t *col_types,
                                uint32_t n_cols, uint32_t R, const uint64_t *cells, const uint8_t *ok, int64_t *out_t,
                                uint8_t *const *out_cells, uint8_t *out_ok, size_t out_rows, int64_t *seg_tmin, int64_t *seg_tmax,
                                unsigned long long *replaced) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= R || !head[i]) return;
    const uint32_t s = row_span[i], local = oidx[i] - out_begin[s], cnt = out_begin[s + 1] - out_begin[s];
    const uint32_t g = seg_base[s] + local / MERGE_RPS, slot = local % MERGE_RPS;
    const size_t dst = (size_t)g * MERGE_RPS + slot;
    const int64_t tt = t[i];
    uint32_t j = i + 1;
    while (j < R && !head[j]) j++;
    if (j - i > 1) atomicAdd(replaced, (unsigned long long)(j - i - 1));
    out_t[dst] = tt;
    for (uint32_t c = 0; c < n_cols; c++) {
        uint64_t v = 0; uint8_t has = 0;
        for (uint32_t k = i; k < j; k++) { /* oldest file first: the last non-null value is the newest one */
            const size_t src = (size_t)c * R + perm[k];
            if (ok[src]) { v = cells[src]; has = 1; }
        }
        out_ok[(size_t)c * out_rows + dst] = has;
        if (col_types[c] == OG_TYPE_BOOL) out_cells[c][dst] = (uint8_t)v;
        else ((uint64_t *)out_cells[c])[dst] = v;
    }
    if (slot == 0) seg_tmin[g] = tt;
    if (slot == MERGE_RPS - 1 || local == cnt - 1) seg_tmax[g] = tt;
}

static SrcDir dir_of(const og_shard *s) {
    SrcDir d;
    d.data = s->d_data; d.page_off = s->d_page_off; d.page_len = s->d_page_len; d.seg_rows = s->d_seg_rows;
    d.n_segments = s->n_segments; d.n_columns = s->n_columns;
    return d;
}

/* a rewritten span: source segments (file order) -> new segments */
struct Span {
    uint32_t series;                 /* union series index */
    std::vector<uint32_t> src;       /* source segments, file-sequence order */
    uint64_t rows = 0;
    uint32_t batch = 0, first_new = 0, n_new = 0; /* new segments [first_new, first_new + n_new) of batch `batch` */
};
struct NewSegs { /* what one batch produced, on the host */
    std::vector<uint64_t> off; std::vector<uint32_t> len; /* [(n_cols+1) * n] relative to the batch blob */
    std::vector<int64_t> tmin, tmax;
    uint8_t *blob = nullptr; uint64_t bytes = 0; uint64_t base = 0; /* blob position in the final data */
    uint32_t n = 0;
};

/* Merge every span on the device, batch by batch.  Fills batches[] and each span's new-segment range. */
static int merge_spans(og_shard *src, const std::vector<Span *> &spans, const std::vector<uint32_t> &src_file, const std::vector<uint64_t> &sids, std::vector<NewSegs> &batches,
                       Scratch &blobs, uint64_t *replaced_out) {
    const uint32_t nc = src->n_columns, ncol1 = nc + 1;
    int rc;
    /* scratch per row: decode (8 t + 4 file + 4 span + 9 per column), sort (4 + 4 perm, 8 keys), heads + scan (8), output slots
       (8 + 9 per column), encoder staging and blob (2 x 8704 / 1000 per page) */
    const uint64_t per_row = 48 + 18ull * nc + 2ull * ncol1 * MERGE_PAGE_BOUND / MERGE_RPS + 64;
    uint64_t cap_rows;
    {
        size_t fr = 0, tot = 0;
        CU(dev_mem_info(&fr, &tot));
        cap_rows = std::max<uint64_t>(MERGE_RPS, (uint64_t)(fr / 4) / per_row);
        if (const char *ov = getenv("OGPU_MERGE_BATCH_ROWS")) cap_rows = std::max<uint64_t>(1, strtoull(ov, nullptr, 10)); /* test hook */
        cap_rows = std::min<uint64_t>(cap_rows, 1ull << 30);
    }
    std::vector<int64_t> h_zero;
    unsigned long long *d_rep; MergeErr *d_err; int32_t *d_types;
    Scratch keep;
    if ((rc = keep.get(&d_rep, 1)) || (rc = keep.get(&d_err, 1)) || (rc = keep.get(&d_types, nc))) return rc;
    CU(cudaMemset(d_rep, 0, 8)); CU(cudaMemset(d_err, 0, sizeof(MergeErr)));
    CU(cudaMemcpy(d_types, src->col_types.data(), nc * 4, cudaMemcpyHostToDevice));
    std::vector<uint32_t> seg_rows(src->n_segments);
    CU(cudaMemcpy(seg_rows.data(), src->d_seg_rows, (size_t)src->n_segments * 4, cudaMemcpyDeviceToHost));
    const SrcDir dir = dir_of(src);
    size_t sp0 = 0;
    while (sp0 < spans.size()) {
        size_t sp1 = sp0; uint64_t R64 = 0;
        while (sp1 < spans.size() && (sp1 == sp0 || R64 + spans[sp1]->rows <= cap_rows)) R64 += spans[sp1++]->rows;
        if (R64 >= 0xffffffffull) { set_error("a rewritten span holds %llu rows (limit 2^32 - 2)", (unsigned long long)R64); return OG_E_UNSUPPORTED; }
        const uint32_t R = (uint32_t)R64, nsp = (uint32_t)(sp1 - sp0);
        /* host lists: source segments of the batch and the first row of every span */
        std::vector<uint32_t> h_seg, h_row0, h_file, h_span, h_span_row0;
        uint32_t row = 0;
        for (uint32_t k = 0; k < nsp; k++) {
            h_span_row0.push_back(row);
            for (uint32_t g : spans[sp0 + k]->src) { h_seg.push_back(g); h_row0.push_back(row); h_file.push_back(src_file[g]); h_span.push_back(k); row += seg_rows[g]; }
        }
        h_span_row0.push_back(row);
        const uint32_t nsrc = (uint32_t)h_seg.size();
        Scratch b;
        uint32_t *d_seg, *d_row0, *d_file, *d_span, *d_span_row0, *row_file, *row_span, *perm_in, *perm, *head, *oidx, *out_begin, *seg_base;
        int64_t *times, *times_sorted; uint64_t *cells; uint8_t *ok;
        if ((rc = b.get(&d_seg, nsrc)) || (rc = b.get(&d_row0, nsrc)) || (rc = b.get(&d_file, nsrc)) || (rc = b.get(&d_span, nsrc)) ||
            (rc = b.get(&d_span_row0, nsp + 1)) || (rc = b.get(&row_file, R)) || (rc = b.get(&row_span, R)) ||
            (rc = b.get(&perm_in, R)) || (rc = b.get(&perm, R)) || (rc = b.get(&head, (size_t)R + 1)) ||
            (rc = b.get(&oidx, (size_t)R + 1)) || (rc = b.get(&out_begin, nsp + 1)) || (rc = b.get(&seg_base, nsp)) ||
            (rc = b.get(&times, R)) || (rc = b.get(&times_sorted, R)) || (rc = b.get(&cells, (size_t)nc * R)) ||
            (rc = b.get(&ok, (size_t)nc * R)))
            return rc;
        CU(cudaMemcpy(d_seg, h_seg.data(), nsrc * 4ull, cudaMemcpyHostToDevice));
        CU(cudaMemcpy(d_row0, h_row0.data(), nsrc * 4ull, cudaMemcpyHostToDevice));
        CU(cudaMemcpy(d_file, h_file.data(), nsrc * 4ull, cudaMemcpyHostToDevice));
        CU(cudaMemcpy(d_span, h_span.data(), nsrc * 4ull, cudaMemcpyHostToDevice));
        CU(cudaMemcpy(d_span_row0, h_span_row0.data(), (nsp + 1) * 4ull, cudaMemcpyHostToDevice));
        k_merge_decode<<<(nsrc + 127) / 128, 128>>>(dir, d_types, nsrc, d_seg, d_row0, d_file, d_span, R, times, row_file, row_span, cells, ok, d_err);
        k_merge_iota<<<(R + 255) / 256, 256>>>(perm_in, R);
        { /* rows of a span by time; stable, so equal times keep file order */
            size_t tb = 0; void *tmp = nullptr;
            CU(cub::DeviceSegmentedSort::StableSortPairs(nullptr, tb, times, times_sorted, perm_in, perm, (int)R, (int)nsp, d_span_row0, d_span_row0 + 1));
            if ((rc = b.get((uint8_t **)&tmp, tb))) return rc;
            CU(cub::DeviceSegmentedSort::StableSortPairs(tmp, tb, times, times_sorted, perm_in, perm, (int)R, (int)nsp, d_span_row0, d_span_row0 + 1));
        }
        /* row_span is constant over a span's rows, so it indexes sorted positions as well as decoded ones */
        k_merge_heads<<<(R + 1 + 255) / 256, 256>>>(times_sorted, perm, row_file, row_span, R, head, d_err);
        {
            size_t tb = 0; void *tmp = nullptr;
            CU(cub::DeviceScan::ExclusiveSum(nullptr, tb, head, oidx, (int)R + 1));
            if ((rc = b.get((uint8_t **)&tmp, tb))) return rc;
            CU(cub::DeviceScan::ExclusiveSum(tmp, tb, head, oidx, (int)R + 1));
        }
        k_merge_span_out<<<(nsp + 1 + 127) / 128, 128>>>(d_span_row0, nsp, oidx, out_begin);
        CU(cudaGetLastError());
        MergeErr he;
        CU(cudaMemcpy(&he, d_err, sizeof he, cudaMemcpyDeviceToHost));
        if (he.code) {
            const unsigned long long sid = (unsigned long long)sids[spans[sp0 + he.span]->series];
            if (he.code == M_STRING) { set_error("series sid %llu: string column \"%s\" has values in a span the merge re-encodes (there is no device string encoder)", sid, src->col_names[he.col].c_str()); return OG_E_UNSUPPORTED; }
            if (he.code == M_REPEAT) { set_error("series sid %llu: time %lld appears twice in file %d inside a merged span", sid, he.time, he.file); return OG_E_CORRUPT; }
            set_error("segment %d of the file set failed to decode (device code %d)", he.seg, he.code);
            return he.code == D_UNSUPPORTED ? OG_E_UNSUPPORTED : OG_E_CORRUPT;
        }
        std::vector<uint32_t> h_out(nsp + 1), h_base(nsp);
        CU(cudaMemcpy(h_out.data(), out_begin, (nsp + 1) * 4ull, cudaMemcpyDeviceToHost));
        NewSegs ns;
        std::vector<uint32_t> h_rows;
        for (uint32_t k = 0; k < nsp; k++) {
            const uint32_t cnt = h_out[k + 1] - h_out[k], nseg = (cnt + MERGE_RPS - 1) / MERGE_RPS;
            Span &sp = *spans[sp0 + k];
            sp.batch = (uint32_t)batches.size(); sp.first_new = ns.n; sp.n_new = nseg;
            h_base[k] = ns.n;
            for (uint32_t g = 0; g < nseg; g++) h_rows.push_back(std::min(MERGE_RPS, cnt - g * MERGE_RPS));
            ns.n += nseg;
        }
        const uint32_t NS = ns.n;
        const size_t out_rows = (size_t)NS * MERGE_RPS;
        int64_t *out_t, *d_tmin, *d_tmax; uint8_t *out_ok; uint32_t *d_rows; uint8_t **d_cols;
        std::vector<uint8_t *> h_cols(nc);
        if ((rc = b.get(&out_t, out_rows)) || (rc = b.get(&out_ok, (size_t)nc * out_rows)) || (rc = b.get(&d_tmin, NS)) ||
            (rc = b.get(&d_tmax, NS)) || (rc = b.get(&d_rows, NS)) || (rc = b.get(&d_cols, nc)))
            return rc;
        for (uint32_t c = 0; c < nc; c++)
            if ((rc = b.get(&h_cols[c], out_rows * (src->col_types[c] == OG_TYPE_BOOL ? 1 : 8)))) return rc;
        CU(cudaMemcpy(d_cols, h_cols.data(), nc * sizeof(uint8_t *), cudaMemcpyHostToDevice));
        CU(cudaMemcpy(seg_base, h_base.data(), nsp * 4ull, cudaMemcpyHostToDevice));
        CU(cudaMemcpy(d_rows, h_rows.data(), NS * 4ull, cudaMemcpyHostToDevice));
        k_merge_combine<<<(R + 127) / 128, 128>>>(times_sorted, perm, row_span, head, oidx, out_begin, seg_base, d_types, nc, R, cells, ok,
                                                   out_t, d_cols, out_ok, out_rows, d_tmin, d_tmax, d_rep);
        CU(cudaGetLastError());
        /* encode every column (string columns: no values inside a span, so no page) */
        uint8_t *blob; uint64_t *d_off; uint32_t *d_len;
        const uint64_t cap = (uint64_t)NS * ncol1 * MERGE_PAGE_BOUND;
        if ((rc = b.get(&blob, cap)) || (rc = b.get(&d_off, (size_t)ncol1 * NS)) || (rc = b.get(&d_len, (size_t)ncol1 * NS))) return rc;
        CU(cudaMemset(d_len, 0, (size_t)ncol1 * NS * 4)); CU(cudaMemset(d_off, 0, (size_t)ncol1 * NS * 8));
        uint64_t used = 0;
        ns.off.assign((size_t)ncol1 * NS, 0); ns.len.assign((size_t)ncol1 * NS, 0);
        for (uint32_t c = 0; c <= nc; c++) {
            const bool is_time = c == nc;
            if (!is_time && src->col_types[c] == OG_TYPE_STRING) continue;
            uint64_t tot = 0;
            rc = encode_pages(is_time ? OG_TYPE_INT : src->col_types[c], is_time ? 1 : 0, is_time ? (const void *)out_t : (const void *)h_cols[c],
                              is_time ? nullptr : out_ok + (size_t)c * out_rows, d_rows, NS, MERGE_RPS, blob + used, cap - used,
                              d_off + (size_t)c * NS, d_len + (size_t)c * NS, &tot, true);
            if (rc) return rc;
            CU(cudaMemcpy(ns.off.data() + (size_t)c * NS, d_off + (size_t)c * NS, NS * 8ull, cudaMemcpyDeviceToHost));
            CU(cudaMemcpy(ns.len.data() + (size_t)c * NS, d_len + (size_t)c * NS, NS * 4ull, cudaMemcpyDeviceToHost));
            for (uint32_t g = 0; g < NS; g++) ns.off[(size_t)c * NS + g] += used;
            used += tot;
        }
        ns.tmin.resize(NS); ns.tmax.resize(NS);
        CU(cudaMemcpy(ns.tmin.data(), d_tmin, NS * 8ull, cudaMemcpyDeviceToHost));
        CU(cudaMemcpy(ns.tmax.data(), d_tmax, NS * 8ull, cudaMemcpyDeviceToHost));
        /* keep only the bytes written: the batch's scratch goes back to the pool before the next batch */
        if ((rc = blobs.get(&ns.blob, used))) return rc;
        CU(cudaMemcpy(ns.blob, blob, used, cudaMemcpyDeviceToDevice));
        ns.bytes = used;
        batches.push_back(std::move(ns));
        sp0 = sp1;
    }
    unsigned long long rep = 0;
    CU(cudaMemcpy(&rep, d_rep, 8, cudaMemcpyDeviceToHost));
    *replaced_out = rep;
    return OG_OK;
}

} // namespace ogpu

using namespace ogpu;

extern "C" {

OG_API int og_shard_open_files(const og_shard_desc *files, const uint32_t *file_flags, uint32_t n_files, og_shard **out) {
    if (!files || !out || n_files == 0) { set_error("null argument or no files"); return OG_E_INVAL; }
    *out = nullptr;
    int rc = ensure_device(); if (rc) return rc;
    int dev = 0; CU(cudaGetDevice(&dev));
    auto is_ooo = [&](uint32_t f) { return file_flags && (file_flags[f] & OG_FILE_OUT_OF_ORDER); };
    /* ---- checks, schema union by name (sorted), series union by sid (ascending) ---- */
    std::map<std::string, int32_t> schema;
    std::map<uint64_t, uint32_t> series_of_sid;
    for (uint32_t f = 0; f < n_files; f++) {
        const og_shard_desc *d = &files[f];
        if (d->flags & OG_SHARD_DEVICE_DATA) { set_error("file %u: OG_SHARD_DEVICE_DATA is not accepted by og_shard_open_files (the files are copied into one buffer)", f); return OG_E_INVAL; }
        if (d->data_len && !d->data) { set_error("file %u: null data", f); return OG_E_INVAL; }
        if ((rc = check_desc(d))) { char m[512]; snprintf(m, sizeof m, "%s", og_last_error()); set_error("file %u: %s", f, m); return rc; }
        std::map<std::string, int> seen;
        for (uint32_t c = 0; c < d->n_columns; c++) {
            const std::string name = d->columns[c].name ? d->columns[c].name : "";
            if (seen.count(name)) { set_error("file %u: column \"%s\" appears twice", f, name.c_str()); return OG_E_INVAL; }
            seen[name] = 1;
            auto it = schema.find(name);
            if (it == schema.end()) schema[name] = d->columns[c].type;
            else if (it->second != d->columns[c].type) { set_error("column \"%s\" has type %d in one file and %d in file %u", name.c_str(), it->second, d->columns[c].type, f); return OG_E_TYPE; }
        }
        std::map<uint64_t, int> sseen;
        for (uint32_t s = 0; s < d->n_series; s++) {
            if (sseen.count(d->sids[s])) { set_error("file %u: sid %llu appears twice", f, (unsigned long long)d->sids[s]); return OG_E_INVAL; }
            sseen[d->sids[s]] = 1;
            series_of_sid[d->sids[s]] = 0;
        }
    }
    if (schema.size() > 64) { set_error("the files hold %zu distinct columns (limit 64)", schema.size()); return OG_E_INVAL; }
    std::vector<std::string> names; std::vector<int32_t> types;
    for (auto &kv : schema) { names.push_back(kv.first); types.push_back(kv.second); }
    std::vector<uint64_t> sids;
    for (auto &kv : series_of_sid) { kv.second = (uint32_t)sids.size(); sids.push_back(kv.first); }
    const uint32_t nc = (uint32_t)names.size(), ncol1 = nc + 1, NSER = (uint32_t)sids.size();
    /* ---- the source directory: every segment of every file, file by file, page offsets rebased into one buffer ---- */
    std::vector<uint64_t> base(n_files), seg0(n_files + 1, 0), ser0(n_files + 1, 0);
    uint64_t data_len = 0;
    for (uint32_t f = 0; f < n_files; f++) {
        base[f] = (data_len + 15) & ~15ull; data_len = base[f] + files[f].data_len;
        seg0[f + 1] = seg0[f] + files[f].n_segments; ser0[f + 1] = ser0[f] + files[f].n_series;
    }
    if (seg0[n_files] > 0xfffffff0ull) { set_error("too many segments"); return OG_E_INVAL; }
    const uint32_t NSRC = (uint32_t)seg0[n_files];
    std::vector<uint64_t> off((size_t)ncol1 * NSRC, 0); std::vector<uint32_t> len((size_t)ncol1 * NSRC, 0);
    std::vector<int64_t> tmin(NSRC), tmax(NSRC);
    std::vector<uint32_t> src_file(NSRC), ssb; ssb.reserve(ser0[n_files] + 1);
    for (uint32_t f = 0; f < n_files; f++) {
        const og_shard_desc *d = &files[f];
        std::vector<int> col_of(d->n_columns);
        for (uint32_t c = 0; c < d->n_columns; c++) col_of[c] = (int)(std::lower_bound(names.begin(), names.end(), std::string(d->columns[c].name ? d->columns[c].name : "")) - names.begin());
        for (uint32_t g = 0; g < d->n_segments; g++) {
            const size_t gs = seg0[f] + g;
            src_file[gs] = f; tmin[gs] = d->seg_tmin[g]; tmax[gs] = d->seg_tmax[g];
            for (uint32_t c = 0; c < d->n_columns; c++)
                if (d->columns[c].page_len[g]) { off[(size_t)col_of[c] * NSRC + gs] = base[f] + d->columns[c].page_off[g]; len[(size_t)col_of[c] * NSRC + gs] = d->columns[c].page_len[g]; }
            off[(size_t)nc * NSRC + gs] = base[f] + d->time_page_off[g]; len[(size_t)nc * NSRC + gs] = d->time_page_len[g];
        }
        for (uint32_t s = 0; s < d->n_series; s++) ssb.push_back((uint32_t)(seg0[f] + d->series_seg_begin[s]));
    }
    ssb.push_back(NSRC);
    /* ---- per series: ordered segments in file order (no overlap across files), out-of-order segments, the span ---- */
    std::vector<std::vector<uint32_t>> ordered(NSER), ooo(NSER);
    std::vector<std::vector<uint32_t>> ord_file(NSER);
    og_merge_info info{}; info.n_files = n_files;
    for (uint32_t f = 0; f < n_files; f++) {
        const og_shard_desc *d = &files[f];
        if (is_ooo(f)) info.n_out_of_order_files++;
        for (uint32_t s = 0; s < d->n_series; s++) {
            const uint32_t u = series_of_sid[d->sids[s]];
            for (uint32_t g = d->series_seg_begin[s]; g < d->series_seg_begin[s + 1]; g++) {
                const uint32_t gs = (uint32_t)(seg0[f] + g);
                if (is_ooo(f)) { ooo[u].push_back(gs); continue; }
                if (!ordered[u].empty() && tmin[gs] <= tmax[ordered[u].back()]) {
                    set_error("series sid %llu: ordered files %u and %u overlap in time (%lld <= %lld); only out-of-order files may overlap",
                              (unsigned long long)sids[u], src_file[ordered[u].back()], f, (long long)tmin[gs], (long long)tmax[ordered[u].back()]);
                    return OG_E_UNSUPPORTED;
                }
                ordered[u].push_back(gs);
            }
        }
    }
    /* layout of the output series: kept ordered segments before the span, the span, kept ones after it */
    std::vector<Span> span_store; span_store.reserve(NSER);
    std::vector<uint32_t> before(NSER), after_begin(NSER);
    std::vector<int> span_of(NSER, -1);
    for (uint32_t u = 0; u < NSER; u++) {
        const auto &o = ordered[u];
        if (ooo[u].empty()) { before[u] = after_begin[u] = (uint32_t)o.size(); continue; }
        int64_t lo = INT64_MAX, hi = INT64_MIN;
        for (uint32_t g : ooo[u]) { lo = std::min(lo, tmin[g]); hi = std::max(hi, tmax[g]); }
        uint32_t a = 0, b;
        while (a < o.size() && tmax[o[a]] < lo) a++;
        b = a;
        while (b < o.size() && tmin[o[b]] <= hi) b++;
        before[u] = a; after_begin[u] = b;
        Span sp; sp.series = u;
        sp.src.assign(o.begin() + a, o.begin() + b);
        sp.src.insert(sp.src.end(), ooo[u].begin(), ooo[u].end());
        /* oldest first: ordered files, then out-of-order files, each in file sequence (every out-of-order file is newer than
           every ordered one, whatever their positions in files[]) */
        auto rank = [&](uint32_t g) { return std::make_pair(is_ooo(src_file[g]) ? 1 : 0, src_file[g]); };
        std::stable_sort(sp.src.begin(), sp.src.end(), [&](uint32_t x, uint32_t y) { return rank(x) < rank(y); });
        span_of[u] = (int)span_store.size();
        span_store.push_back(std::move(sp));
    }
    /* ---- upload (one H2D per file), validate + transcode Snappy over the whole file set ---- */
    std::unique_ptr<og_shard> src(new og_shard);
    src->device = dev; src->n_series = (uint32_t)ser0[n_files]; src->n_segments = NSRC; src->n_columns = nc;
    src->col_types = types; src->col_names = names; src->data_len = data_len;
    src->h_series_seg_begin = ssb;
    for (uint32_t f = 0; f < n_files; f++) src->sids.insert(src->sids.end(), files[f].sids, files[f].sids + files[f].n_series);
    if ((rc = dalloc(&src->d_data, data_len + 1024))) return rc;
    CU(cudaMemset(src->d_data, 0, data_len + 1024));
    for (uint32_t f = 0; f < n_files; f++)
        if (files[f].data_len) CU(cudaMemcpy(src->d_data + base[f], files[f].data, files[f].data_len, cudaMemcpyHostToDevice));
    if ((rc = upload_dir(src.get(), ssb.data(), tmin.data(), tmax.data(), off.data(), len.data(), src->sids.data()))) return rc;
    if ((rc = shard_finalize(src.get(), true))) return rc;
    /* the transcoded directory and the row counts */
    CU(cudaMemcpy(off.data(), src->d_page_off, off.size() * 8, cudaMemcpyDeviceToHost));
    CU(cudaMemcpy(len.data(), src->d_page_len, len.size() * 4, cudaMemcpyDeviceToHost));
    {
        std::vector<uint32_t> rows(NSRC);
        CU(cudaMemcpy(rows.data(), src->d_seg_rows, NSRC * 4ull, cudaMemcpyDeviceToHost));
        for (auto &sp : span_store) {
            for (uint32_t g : sp.src) sp.rows += rows[g];
            info.series_merged++;
            info.segments_rewritten_in += sp.src.size();
        }
        for (uint32_t u = 0; u < NSER; u++) for (uint32_t g : ooo[u]) info.out_of_order_rows += rows[g];
    }
    /* ---- device merge ---- */
    std::vector<NewSegs> batches;
    Scratch blobs; /* the pages of every batch, until they are copied into the output data */
    cudaEvent_t ev0, ev1;
    CU(cudaEventCreate(&ev0)); CU(cudaEventCreate(&ev1));
    struct FreeEv { cudaEvent_t a, b; ~FreeEv() { cudaEventDestroy(a); cudaEventDestroy(b); } } free_ev{ev0, ev1};
    CU(cudaEventRecord(ev0, 0));
    {
        std::vector<Span *> sp;
        for (auto &x : span_store) sp.push_back(&x);
        uint64_t replaced = 0;
        if ((rc = merge_spans(src.get(), sp, src_file, sids, batches, blobs, &replaced))) return rc;
        info.rows_replaced = replaced;
    }
    /* ---- final data: the file set's bytes, then the new pages of every batch ---- */
    uint64_t new_len = src->data_len;
    for (auto &b : batches) { b.base = (new_len + 15) & ~15ull; new_len = b.base + b.bytes; }
    std::unique_ptr<og_shard> s(new og_shard);
    s->device = dev; s->n_series = NSER; s->n_columns = nc; s->col_types = types; s->col_names = names; s->sids = sids;
    if (batches.empty()) { s->d_data = src->d_data; src->d_data = nullptr; s->data_len = src->data_len; }
    else {
        if ((rc = dalloc(&s->d_data, new_len + 1024))) return rc;
        s->data_len = new_len;
        CU(cudaMemset(s->d_data, 0, new_len + 1024));
        CU(cudaMemcpy(s->d_data, src->d_data, src->data_len, cudaMemcpyDeviceToDevice));
        for (auto &b : batches) if (b.bytes) CU(cudaMemcpy(s->d_data + b.base, b.blob, b.bytes, cudaMemcpyDeviceToDevice));
    }
    CU(cudaEventRecord(ev1, 0));
    if (batches.empty()) { s->snappy_pages = src->snappy_pages; s->snappy_bytes_in = src->snappy_bytes_in; s->snappy_bytes_out = src->snappy_bytes_out; }
    src.reset();
    /* ---- the output directory ---- */
    std::vector<uint32_t> o_ssb(NSER + 1, 0);
    std::vector<uint64_t> o_off; std::vector<uint32_t> o_len; std::vector<int64_t> o_tmin, o_tmax;
    struct Ref { int batch; uint32_t seg; }; /* batch < 0: source segment */
    std::vector<Ref> refs;
    for (uint32_t u = 0; u < NSER; u++) {
        o_ssb[u] = (uint32_t)refs.size();
        const auto &o = ordered[u];
        for (uint32_t i = 0; i < before[u]; i++) refs.push_back({-1, o[i]});
        if (span_of[u] >= 0) { const Span &sp = span_store[span_of[u]]; for (uint32_t g = 0; g < sp.n_new; g++) refs.push_back({(int)sp.batch, sp.first_new + g}); }
        for (uint32_t i = after_begin[u]; i < o.size(); i++) refs.push_back({-1, o[i]});
        info.segments_kept += before[u] + (o.size() - after_begin[u]);
    }
    const uint32_t NOUT = (uint32_t)refs.size();
    o_ssb[NSER] = NOUT;
    o_off.resize((size_t)ncol1 * NOUT); o_len.resize((size_t)ncol1 * NOUT); o_tmin.resize(NOUT); o_tmax.resize(NOUT);
    for (uint32_t i = 0; i < NOUT; i++) {
        const Ref r = refs[i];
        for (uint32_t c = 0; c < ncol1; c++) {
            if (r.batch < 0) { o_off[(size_t)c * NOUT + i] = off[(size_t)c * NSRC + r.seg]; o_len[(size_t)c * NOUT + i] = len[(size_t)c * NSRC + r.seg]; }
            else {
                const NewSegs &b = batches[r.batch];
                const uint32_t l = b.len[(size_t)c * b.n + r.seg];
                o_off[(size_t)c * NOUT + i] = l ? b.base + b.off[(size_t)c * b.n + r.seg] : 0; o_len[(size_t)c * NOUT + i] = l;
            }
        }
        if (r.batch < 0) { o_tmin[i] = tmin[r.seg]; o_tmax[i] = tmax[r.seg]; }
        else { o_tmin[i] = batches[r.batch].tmin[r.seg]; o_tmax[i] = batches[r.batch].tmax[r.seg]; }
        info.segments_rewritten_out += r.batch >= 0;
    }
    s->n_segments = NOUT; s->h_series_seg_begin = o_ssb;
    s->tmin = INT64_MAX; s->tmax = INT64_MIN;
    for (uint32_t i = 0; i < NOUT; i++) { s->tmin = std::min(s->tmin, o_tmin[i]); s->tmax = std::max(s->tmax, o_tmax[i]); }
    if ((rc = upload_dir(s.get(), o_ssb.data(), o_tmin.data(), o_tmax.data(), o_off.data(), o_len.data(), sids.data()))) return rc;
    if ((rc = shard_finalize(s.get(), false))) return rc;
    float ms = 0;
    CU(cudaEventElapsedTime(&ms, ev0, ev1));
    info.merge_ms = ms;
    info.rows_after_merge = s->n_rows;
    s->merge = info;
    *out = s.release();
    return OG_OK;
}

OG_API int og_shard_merge_info(const og_shard *s, og_merge_info *out) {
    if (!s || !out) { set_error("null argument"); return OG_E_INVAL; }
    *out = s->merge;
    return OG_OK;
}

} // extern "C"
