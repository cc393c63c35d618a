/*
 * merge.cu — TSSP files into a shard (DESIGN.md (d) "Bringing files into a shard").  og_shard_open_files opens the ordered and
 * out-of-order files of one shard as ONE og_shard; og_shard_append_files adds files flushed into an open shard.  An open is an
 * append to an empty shard: both run add_files.  add_files takes new files from one of two producers: upload_files (host files
 * copied in, validated, transcoded) or place_files (the files og_shard_append_rows encoded on the device, flush.cu); everything
 * from the probe on is one path for both.
 *
 * The reference merges a shard's files for every series of every query (include/ogpu.h lists the code).  Here the merge runs
 * once, when the files join the shard:
 *
 *   host   check every description (check_desc), union of columns by name and of series by sid with the shard's, the ordered
 *          segments of a series in file order (overlapping ordered files are refused), one H2D per file into one data buffer with
 *          rebased page offsets; the new files are validated and their Snappy pages transcoded by shard_finalize, so the merge only
 *          sees codecs ColIter / TimeIter decode.  The shard's own pages are not validated again.
 *   probe  k_append_probe: per series of the shard that takes new segments, its last time (a new ordered segment must start after
 *          it) and the range of its segments a span overlaps.
 *   order  the rows of one time are ranked oldest first: the shard's rows, then ordered files, then out-of-order files, each in
 *          file sequence.
 *   span   per series with out-of-order rows: the hull [min, max] of its out-of-order segments' time ranges, widened to the shard's
 *          and the new ordered segments it overlaps.  Those segments and every out-of-order segment of the series are rewritten;
 *          every other segment keeps its bytes.
 *   device the spans' source segments spliced into one directory (k_append_splice, k_append_gather), then per batch of spans
 *          (scratch ~ rows in the batch, under a device-memory budget):
 *          k_merge_decode   one thread per source segment: rows of every union column, laid out span by span, sources of a span
 *                           in file-sequence order
 *          StableSortPairs  by time inside each span (cub segmented sort): rows of equal time stay in file order, oldest first
 *          k_merge_heads    first row of each run of equal times; a time repeated inside one file is OG_E_CORRUPT
 *          k_merge_combine  one thread per run: each column takes its newest non-null value (mergeRecRow, record.go:468-505),
 *                           written into 1000-row segment slots (lib/util/util.go:72)
 *          encode_pages     the adaptive encoders of og_encode_pages (encode.cu), raw page for a float segment Gorilla refuses
 *   finish k_append_splice builds the new directory from runs of the shard's, the files' and the merge's segments; k_append_gather
 *          copies the live pages into a new data region, unless the files' region already holds every one of them (nothing merged
 *          and no older segments), which is then kept as it is; k_append_stats derives the shard's totals from the time pages'
 *          headers, and install_state swaps the new state in whole.
 *
 * The gather's copy loop is not shared with k_tssp_gather: the writer's CRC needs each lane to own one contiguous slice of a page,
 * the gather deals 16-byte blocks out across the lanes so that a warp's loads and stores are consecutive.
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
#include "span_pass.h"

namespace ogpu {

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

/* one thread per run of equal times: the row rule, then the merged row into its 1000-row segment slot.  span_has (may be null):
 * [span][column] set where the column holds a value in the span */
__global__ void k_merge_combine(const int64_t *t, const uint32_t *perm, const uint32_t *row_span, const uint32_t *head,
                                const uint32_t *oidx, const uint32_t *out_begin, const uint32_t *seg_base, const int32_t *col_types,
                                uint32_t n_cols, uint32_t R, const uint64_t *cells, const uint8_t *ok, int64_t *out_t,
                                uint8_t *const *out_cells, uint8_t *out_ok, size_t out_rows, int64_t *seg_tmin, int64_t *seg_tmax,
                                unsigned long long *replaced, uint8_t *span_has) {
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
        if (has && span_has) span_has[(size_t)s * n_cols + c] = 1;
        if (col_types[c] == OG_TYPE_BOOL) out_cells[c][dst] = (uint8_t)v;
        else ((uint64_t *)out_cells[c])[dst] = v;
    }
    if (slot == 0) seg_tmin[g] = tt;
    if (slot == MERGE_RPS - 1 || local == cnt - 1) seg_tmax[g] = tt;
}

/* a rewritten span: source segments (file order) -> new segments */
struct Span {
    uint32_t series;                 /* union series index */
    std::vector<uint32_t> src;       /* source segments, file-sequence order */
    std::vector<uint32_t> src_file, src_rows; /* per source segment: its file (one file never repeats a time) and its rows */
    uint64_t rows = 0;
    uint32_t batch = 0, first_new = 0, n_new = 0; /* new segments [first_new, first_new + n_new) of batch `batch` */
};

/* ---------------------------------------------------------------- sort, runs and the row rule (shared with the flush) */

int sort_spans(const int64_t *times, int64_t *times_sorted, uint32_t *perm_in, uint32_t *perm, uint32_t R, uint32_t n_spans,
               const uint32_t *d_span_row0, Scratch &b) {
    int rc;
    k_merge_iota<<<(R + 255) / 256, 256>>>(perm_in, R);
    size_t tb = 0; void *tmp = nullptr;
    CU(cub::DeviceSegmentedSort::StableSortPairs(nullptr, tb, times, times_sorted, perm_in, perm, (int)R, (int)n_spans, d_span_row0, d_span_row0 + 1));
    if ((rc = b.get((uint8_t **)&tmp, tb))) return rc;
    CU(cub::DeviceSegmentedSort::StableSortPairs(tmp, tb, times, times_sorted, perm_in, perm, (int)R, (int)n_spans, d_span_row0, d_span_row0 + 1));
    return OG_OK;
}

int find_runs(SortedRows &r, const uint32_t *row_file, Scratch &b, MergeErr *d_err) {
    int rc;
    if ((rc = b.get(&r.head, (size_t)r.R + 1)) || (rc = b.get(&r.oidx, (size_t)r.R + 1)) || (rc = b.get(&r.out_begin, r.n_spans + 1))) return rc;
    k_merge_heads<<<(r.R + 1 + 255) / 256, 256>>>(r.t, r.perm, row_file, r.row_span, r.R, r.head, d_err);
    {
        size_t tb = 0; void *tmp = nullptr;
        CU(cub::DeviceScan::ExclusiveSum(nullptr, tb, r.head, r.oidx, (int)r.R + 1));
        if ((rc = b.get((uint8_t **)&tmp, tb))) return rc;
        CU(cub::DeviceScan::ExclusiveSum(tmp, tb, r.head, r.oidx, (int)r.R + 1));
    }
    k_merge_span_out<<<(r.n_spans + 1 + 127) / 128, 128>>>(r.span_row0, r.n_spans, r.oidx, r.out_begin);
    CU(cudaGetLastError());
    return OG_OK;
}

int combine_and_encode(const SortedRows &r, const std::vector<int32_t> &types, const int32_t *d_types, Scratch &b, unsigned long long *d_rep,
                       uint8_t *span_has, Scratch &blobs, NewSegs &ns, std::vector<uint32_t> &seg_first) {
    int rc;
    const uint32_t nc = (uint32_t)types.size(), ncol1 = nc + 1, nsp = r.n_spans;
    std::vector<uint32_t> h_out(nsp + 1), h_rows;
    CU(cudaMemcpy(h_out.data(), r.out_begin, (nsp + 1) * 4ull, cudaMemcpyDeviceToHost));
    seg_first.assign(nsp + 1, 0);
    for (uint32_t k = 0; k < nsp; k++) {
        const uint32_t cnt = h_out[k + 1] - h_out[k], nseg = (cnt + MERGE_RPS - 1) / MERGE_RPS;
        seg_first[k + 1] = seg_first[k] + nseg;
        for (uint32_t g = 0; g < nseg; g++) h_rows.push_back(std::min(MERGE_RPS, cnt - g * MERGE_RPS));
    }
    const uint32_t NS = ns.n = seg_first[nsp];
    const size_t out_rows = (size_t)NS * MERGE_RPS;
    int64_t *out_t, *d_tmin, *d_tmax; uint8_t *out_ok; uint32_t *d_rows, *seg_base; uint8_t **d_cols;
    std::vector<uint8_t *> h_cols(nc);
    if ((rc = b.get(&out_t, out_rows)) || (rc = b.get(&out_ok, (size_t)nc * out_rows)) || (rc = b.get(&d_tmin, NS)) ||
        (rc = b.get(&d_tmax, NS)) || (rc = b.get(&d_rows, NS)) || (rc = b.get(&d_cols, nc)) || (rc = b.get(&seg_base, nsp)))
        return rc;
    for (uint32_t c = 0; c < nc; c++)
        if ((rc = b.get(&h_cols[c], out_rows * (types[c] == OG_TYPE_BOOL ? 1 : 8)))) return rc;
    CU(cudaMemcpy(d_cols, h_cols.data(), nc * sizeof(uint8_t *), cudaMemcpyHostToDevice));
    CU(cudaMemcpy(seg_base, seg_first.data(), nsp * 4ull, cudaMemcpyHostToDevice));
    CU(cudaMemcpy(d_rows, h_rows.data(), NS * 4ull, cudaMemcpyHostToDevice));
    k_merge_combine<<<(r.R + 127) / 128, 128>>>(r.t, r.perm, r.row_span, r.head, r.oidx, r.out_begin, seg_base, d_types, nc, r.R, r.cells, r.ok,
                                                 out_t, d_cols, out_ok, out_rows, d_tmin, d_tmax, d_rep, span_has);
    CU(cudaGetLastError());
    /* encode every column (string columns: no values inside a span, so no page) */
    uint8_t *blob;
    const uint64_t cap = (uint64_t)NS * ncol1 * MERGE_PAGE_BOUND;
    if ((rc = b.get(&blob, cap))) return rc;
    uint64_t used = 0;
    if ((rc = encode_columns(types, out_t, h_cols, out_ok, out_rows, d_rows, NS, MERGE_RPS, blob, cap, ns, &used))) return rc;
    return keep_blob(d_tmin, d_tmax, std::move(h_rows), blob, used, blobs, ns);
}

/* Merge every span on the device, batch by batch: the spans' source segments are read through `dir`, whose columns are `types` /
 * `names` and whose segments `dir_runs` spliced from the shard and the files.  Fills batches[] and each span's new-segment range.
 * A repeated time names its file, or the shard's rows when the file is `shard_file`.  Every batch's blob is followed by 1024
 * readable bytes (k_append_gather reads past a page's end). */
static int merge_spans(const SrcDir &dir, const std::vector<Run> &dir_runs, const std::vector<int32_t> &types, const std::vector<std::string> &names,
                       const std::vector<Span *> &spans, const std::vector<uint64_t> &sids, uint32_t shard_file, std::vector<NewSegs> &batches,
                       Scratch &blobs, uint64_t *replaced_out) {
    const uint32_t nc = dir.n_columns;
    int rc;
    uint64_t cap_rows;
    if ((rc = batch_cap_rows(span_row_bytes(nc), MERGE_RPS, "OGPU_MERGE_BATCH_ROWS", &cap_rows))) return rc;
    unsigned long long *d_rep; MergeErr *d_err; int32_t *d_types;
    Scratch keep;
    if ((rc = keep.get(&d_rep, 1)) || (rc = keep.get(&d_err, 1)) || (rc = keep.get(&d_types, nc))) return rc;
    CU(cudaMemset(d_rep, 0, 8)); CU(cudaMemset(d_err, 0, sizeof(MergeErr)));
    CU(cudaMemcpy(d_types, types.data(), nc * 4, cudaMemcpyHostToDevice));
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
            const Span &sp = *spans[sp0 + k];
            for (size_t j = 0; j < sp.src.size(); j++) { h_seg.push_back(sp.src[j]); h_row0.push_back(row); h_file.push_back(sp.src_file[j]); h_span.push_back(k); row += sp.src_rows[j]; }
        }
        h_span_row0.push_back(row);
        const uint32_t nsrc = (uint32_t)h_seg.size();
        Scratch b;
        uint32_t *d_seg, *d_row0, *d_file, *d_span, *d_span_row0, *row_file, *row_span, *perm_in, *perm;
        int64_t *times, *times_sorted; uint64_t *cells; uint8_t *ok;
        if ((rc = b.get(&d_seg, nsrc)) || (rc = b.get(&d_row0, nsrc)) || (rc = b.get(&d_file, nsrc)) || (rc = b.get(&d_span, nsrc)) ||
            (rc = b.get(&d_span_row0, nsp + 1)) || (rc = b.get(&row_file, R)) || (rc = b.get(&row_span, R)) ||
            (rc = b.get(&perm_in, R)) || (rc = b.get(&perm, R)) || (rc = b.get(&times, R)) || (rc = b.get(&times_sorted, R)) ||
            (rc = b.get(&cells, (size_t)nc * R)) || (rc = b.get(&ok, (size_t)nc * R)))
            return rc;
        CU(cudaMemcpy(d_seg, h_seg.data(), nsrc * 4ull, cudaMemcpyHostToDevice));
        CU(cudaMemcpy(d_row0, h_row0.data(), nsrc * 4ull, cudaMemcpyHostToDevice));
        CU(cudaMemcpy(d_file, h_file.data(), nsrc * 4ull, cudaMemcpyHostToDevice));
        CU(cudaMemcpy(d_span, h_span.data(), nsrc * 4ull, cudaMemcpyHostToDevice));
        CU(cudaMemcpy(d_span_row0, h_span_row0.data(), (nsp + 1) * 4ull, cudaMemcpyHostToDevice));
        k_merge_decode<<<(nsrc + 127) / 128, 128>>>(dir, d_types, nsrc, d_seg, d_row0, d_file, d_span, R, times, row_file, row_span, cells, ok, d_err);
        /* rows of a span by time; stable, so equal times keep file order */
        if ((rc = sort_spans(times, times_sorted, perm_in, perm, R, nsp, d_span_row0, b))) return rc;
        /* row_span is constant over a span's rows, so it indexes sorted positions as well as decoded ones */
        SortedRows sr{times_sorted, perm, row_span, d_span_row0, cells, ok, R, nsp};
        if ((rc = find_runs(sr, row_file, b, d_err))) return rc;
        MergeErr he;
        CU(cudaMemcpy(&he, d_err, sizeof he, cudaMemcpyDeviceToHost));
        if (he.code) {
            const unsigned long long sid = (unsigned long long)sids[spans[sp0 + he.span]->series];
            if (he.code == M_STRING) return string_refusal(sid, names[he.col], "the merge");
            if (he.code == M_REPEAT && (uint32_t)he.file == shard_file) { set_error("series sid %llu: time %lld appears twice in the shard's rows inside a merged span", sid, he.time); return OG_E_CORRUPT; }
            if (he.code == M_REPEAT) { set_error("series sid %llu: time %lld appears twice in file %d inside a merged span", sid, he.time, he.file); return OG_E_CORRUPT; }
            const Run &r = *std::prev(std::upper_bound(dir_runs.begin(), dir_runs.end(), (uint32_t)he.seg, [](uint32_t g, const Run &x) { return g < x.out0; }));
            return decode_failure(he.code, r.src0 + ((uint32_t)he.seg - r.out0), r.kind == SRC_SHARD ? "shard" : "file set");
        }
        NewSegs ns;
        std::vector<uint32_t> seg_first;
        if ((rc = combine_and_encode(sr, types, d_types, b, d_rep, nullptr, blobs, ns, seg_first))) return rc;
        for (uint32_t k = 0; k < nsp; k++) {
            Span &sp = *spans[sp0 + k];
            sp.batch = (uint32_t)batches.size(); sp.first_new = seg_first[k]; sp.n_new = seg_first[k + 1] - seg_first[k];
        }
        batches.push_back(std::move(ns));
        sp0 = sp1;
    }
    unsigned long long rep = 0;
    CU(cudaMemcpy(&rep, d_rep, 8, cudaMemcpyDeviceToHost));
    *replaced_out = rep;
    return OG_OK;
}

/* The checks of every file description and the unions of a file set: columns by name (a column with two types is OG_E_TYPE) and
 * series by sid.  `schema` may hold the columns of a shard the files join. */
static int scan_files(const og_shard_desc *files, uint32_t n_files, const char *who, std::map<std::string, int32_t> &schema,
                      std::map<uint64_t, uint32_t> &series_of_sid) {
    int rc;
    for (uint32_t f = 0; f < n_files; f++) {
        const og_shard_desc *d = &files[f];
        if (d->flags & OG_SHARD_DEVICE_DATA) { set_error("file %u: OG_SHARD_DEVICE_DATA is not accepted by %s (the files are copied into one buffer)", f, who); return OG_E_INVAL; }
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
    return OG_OK;
}

/* every segment of every file, file by file, as one source directory over the union columns `names`; page offsets rebased into
 * one buffer (file f at base[f]) */
struct FileDir {
    std::vector<uint64_t> base, seg0, ser0;
    uint64_t data_len = 0;
    uint32_t n = 0; /* segments */
    std::vector<uint64_t> off; std::vector<uint32_t> len; /* [(n_columns + 1) * n], time last */
    std::vector<int64_t> tmin, tmax;
    std::vector<uint32_t> src_file, ssb; /* per segment: its file; per file series: its first segment */
};
static int build_file_dir(const og_shard_desc *files, uint32_t n_files, const std::vector<std::string> &names, FileDir &fd) {
    const uint32_t nc = (uint32_t)names.size(), ncol1 = nc + 1;
    fd.base.assign(n_files, 0); fd.seg0.assign(n_files + 1, 0); fd.ser0.assign(n_files + 1, 0);
    uint64_t data_len = 0;
    for (uint32_t f = 0; f < n_files; f++) {
        fd.base[f] = (data_len + 15) & ~15ull; data_len = fd.base[f] + files[f].data_len;
        fd.seg0[f + 1] = fd.seg0[f] + files[f].n_segments; fd.ser0[f + 1] = fd.ser0[f] + files[f].n_series;
    }
    if (fd.seg0[n_files] > 0xfffffff0ull) { set_error("too many segments"); return OG_E_INVAL; }
    fd.data_len = data_len;
    const uint32_t NSRC = fd.n = (uint32_t)fd.seg0[n_files];
    fd.off.assign((size_t)ncol1 * NSRC, 0); fd.len.assign((size_t)ncol1 * NSRC, 0);
    fd.tmin.resize(NSRC); fd.tmax.resize(NSRC);
    fd.src_file.resize(NSRC); fd.ssb.clear(); fd.ssb.reserve(fd.ser0[n_files] + 1);
    for (uint32_t f = 0; f < n_files; f++) {
        const og_shard_desc *d = &files[f];
        std::vector<int> col_of(d->n_columns);
        for (uint32_t c = 0; c < d->n_columns; c++) col_of[c] = (int)(std::lower_bound(names.begin(), names.end(), std::string(d->columns[c].name ? d->columns[c].name : "")) - names.begin());
        for (uint32_t g = 0; g < d->n_segments; g++) {
            const size_t gs = fd.seg0[f] + g;
            fd.src_file[gs] = f; fd.tmin[gs] = d->seg_tmin[g]; fd.tmax[gs] = d->seg_tmax[g];
            for (uint32_t c = 0; c < d->n_columns; c++)
                if (d->columns[c].page_len[g]) { fd.off[(size_t)col_of[c] * NSRC + gs] = fd.base[f] + d->columns[c].page_off[g]; fd.len[(size_t)col_of[c] * NSRC + gs] = d->columns[c].page_len[g]; }
            fd.off[(size_t)nc * NSRC + gs] = fd.base[f] + d->time_page_off[g]; fd.len[(size_t)nc * NSRC + gs] = d->time_page_len[g];
        }
        for (uint32_t s = 0; s < d->n_series; s++) fd.ssb.push_back((uint32_t)(fd.seg0[f] + d->series_seg_begin[s]));
    }
    fd.ssb.push_back(NSRC);
    return OG_OK;
}

/* the new files' shard: the directory of build_file_dir over the union columns, on the device */
static int new_files_shard(const og_shard_desc *files, uint32_t n_files, const std::vector<std::string> &names, const std::vector<int32_t> &types,
                           int dev, const FileDir &fd, std::unique_ptr<og_shard> &out) {
    out.reset(new og_shard);
    og_shard *src = out.get();
    src->device = dev; src->n_series = (uint32_t)fd.ser0[n_files]; src->n_segments = fd.n; src->n_columns = (uint32_t)names.size();
    src->col_types = types; src->col_names = names; src->data_len = fd.data_len;
    src->h_series_seg_begin = fd.ssb;
    for (uint32_t f = 0; f < n_files; f++) src->sids.insert(src->sids.end(), files[f].sids, files[f].sids + files[f].n_series);
    return upload_dir(src, fd.ssb.data(), fd.tmin.data(), fd.tmax.data(), fd.off.data(), fd.len.data(), src->sids.data());
}

/* one producer of new files on the device: the files' bytes in one device buffer (one H2D per file) under the directory of
 * build_file_dir, validated and with their Snappy pages transcoded (shard_finalize); fd.off / fd.len are updated to the transcoded
 * directory, rows[] gets every segment's rows */
static int upload_files(const og_shard_desc *files, uint32_t n_files, const std::vector<std::string> &names, const std::vector<int32_t> &types,
                        int dev, FileDir &fd, std::unique_ptr<og_shard> &out, std::vector<uint32_t> &rows) {
    int rc;
    std::unique_ptr<og_shard> src;
    if ((rc = new_files_shard(files, n_files, names, types, dev, fd, src))) return rc;
    if ((rc = dalloc(&src->d_data, fd.data_len + 1024))) return rc;
    CU(cudaMemset(src->d_data, 0, fd.data_len + 1024));
    for (uint32_t f = 0; f < n_files; f++)
        if (files[f].data_len) CU(cudaMemcpy(src->d_data + fd.base[f], files[f].data, files[f].data_len, cudaMemcpyHostToDevice));
    if ((rc = shard_finalize(src.get(), true))) return rc;
    CU(cudaMemcpy(fd.off.data(), src->d_page_off, fd.off.size() * 8, cudaMemcpyDeviceToHost));
    CU(cudaMemcpy(fd.len.data(), src->d_page_len, fd.len.size() * 4, cudaMemcpyDeviceToHost));
    rows.resize(fd.n);
    CU(cudaMemcpy(rows.data(), src->d_seg_rows, fd.n * 4ull, cudaMemcpyDeviceToHost));
    out = std::move(src);
    return OG_OK;
}

/* the other producer: files the flush encoded on the device (DeviceFiles), taken over as they lie */
static int place_files(const og_shard_desc *files, uint32_t n_files, const std::vector<std::string> &names, const std::vector<int32_t> &types,
                       int dev, const FileDir &fd, DeviceFiles &df, std::unique_ptr<og_shard> &out, std::vector<uint32_t> &rows) {
    int rc;
    if (df.data_len < fd.data_len || df.rows.size() != fd.n) { set_error("internal: the device files do not match their directory"); return OG_E_INVAL; }
    std::unique_ptr<og_shard> src;
    if ((rc = new_files_shard(files, n_files, names, types, dev, fd, src))) return rc;
    if ((rc = dalloc(&src->d_seg_rows, fd.n))) return rc;
    CU(cudaMemcpy(src->d_seg_rows, df.rows.data(), fd.n * 4ull, cudaMemcpyHostToDevice));
    src->d_data = df.data; df.data = nullptr;
    rows = df.rows;
    out = std::move(src);
    return OG_OK;
}

static bool file_is_ooo(const uint32_t *file_flags, uint32_t f) { return file_flags && (file_flags[f] & OG_FILE_OUT_OF_ORDER); }

/* per union series u: the files' ordered segments in file order and their out-of-order segments; ordered files that overlap in
 * time for one series are OG_E_UNSUPPORTED.  Counts the out-of-order files into `info`. */
static int split_segments(const og_shard_desc *files, uint32_t n_files, const uint32_t *file_flags, const FileDir &fd,
                          std::map<uint64_t, uint32_t> &series_of_sid, const std::vector<uint64_t> &sids,
                          std::vector<std::vector<uint32_t>> &ordered, std::vector<std::vector<uint32_t>> &ooo, og_merge_info &info) {
    for (uint32_t f = 0; f < n_files; f++) {
        const og_shard_desc *d = &files[f];
        const bool late = file_is_ooo(file_flags, f);
        if (late) info.n_out_of_order_files++;
        for (uint32_t s = 0; s < d->n_series; s++) {
            const uint32_t u = series_of_sid[d->sids[s]];
            for (uint32_t g = d->series_seg_begin[s]; g < d->series_seg_begin[s + 1]; g++) {
                const uint32_t gs = (uint32_t)(fd.seg0[f] + g);
                if (late) { ooo[u].push_back(gs); continue; }
                if (!ordered[u].empty() && fd.tmin[gs] <= fd.tmax[ordered[u].back()]) {
                    set_error("series sid %llu: ordered files %u and %u overlap in time (%lld <= %lld); only out-of-order files may overlap",
                              (unsigned long long)sids[u], fd.src_file[ordered[u].back()], f, (long long)fd.tmin[gs], (long long)fd.tmax[ordered[u].back()]);
                    return OG_E_UNSUPPORTED;
                }
                ordered[u].push_back(gs);
            }
        }
    }
    return OG_OK;
}

/* the hull [lo, hi] of a series' out-of-order segments */
static void span_hull(const std::vector<uint32_t> &ooo, const FileDir &fd, int64_t *lo, int64_t *hi) {
    *lo = INT64_MAX; *hi = INT64_MIN;
    for (uint32_t g : ooo) { *lo = std::min(*lo, fd.tmin[g]); *hi = std::max(*hi, fd.tmax[g]); }
}

/* [a, b): the segments of a time-ordered list that [lo, hi] overlaps */
static void span_bounds(const std::vector<uint32_t> &o, const FileDir &fd, int64_t lo, int64_t hi, uint32_t *a, uint32_t *b) {
    uint32_t i = 0;
    while (i < o.size() && fd.tmax[o[i]] < lo) i++;
    *a = i;
    while (i < o.size() && fd.tmin[o[i]] <= hi) i++;
    *b = i;
}

/* oldest first: ordered files, then out-of-order files, each in file sequence (every out-of-order file is newer than every
   ordered one, whatever their positions in files[]) */
static void sort_oldest_first(std::vector<uint32_t> &segs, const FileDir &fd, const uint32_t *file_flags) {
    auto rank = [&](uint32_t g) { return std::make_pair(file_is_ooo(file_flags, fd.src_file[g]) ? 1 : 0, fd.src_file[g]); };
    std::stable_sort(segs.begin(), segs.end(), [&](uint32_t x, uint32_t y) { return rank(x) < rank(y); });
}

/* ---------------------------------------------------------------- the splice */

struct SpliceP {
    SegSrc src[3];
    const Run *runs; uint32_t n_runs, n_out, n_columns;
    uint64_t *off; uint32_t *len, *rows, *series, *region; int64_t *tmin, *tmax; /* the output directory, [(n_columns + 1) * n_out] */
};

/* thread per output segment: its run, then its entries copied from the source, columns remapped (time column last) */
__global__ void k_append_splice(SpliceP p) {
    const uint32_t g = blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= p.n_out) return;
    uint32_t lo = 0, hi = p.n_runs;
    while (hi - lo > 1) { const uint32_t m = (lo + hi) / 2; if (p.runs[m].out0 <= g) lo = m; else hi = m; }
    const Run r = p.runs[lo];
    const SegSrc &S = p.src[r.kind];
    const uint32_t i = r.src0 + (g - r.out0);
    p.tmin[g] = S.tmin[i]; p.tmax[g] = S.tmax[i]; p.rows[g] = S.rows[i]; p.series[g] = r.series;
    p.region[g] = S.seg_region ? S.seg_region[i] : S.region;
    for (uint32_t c = 0; c <= p.n_columns; c++) {
        const int sc = c == p.n_columns ? (int)S.n_columns : S.col ? S.col[c] : (int)c;
        const size_t o = (size_t)c * p.n_out + g;
        if (sc < 0) { p.off[o] = 0; p.len[o] = 0; continue; }
        const size_t pi = (size_t)sc * S.n_segments + i;
        p.off[o] = S.off[pi]; p.len[o] = S.len[pi];
    }
}

/* sizes[n_pages] = 0, so the exclusive scan ends in the total */
__global__ void k_append_sizes(const uint32_t *len, uint64_t n_pages, uint64_t *sizes) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i <= n_pages) sizes[i] = i < n_pages ? len[i] : 0;
}

constexpr int APPEND_GATHER_THREADS = 256;
/* warp per page: the page from its region to its place in the new data region; dst_off becomes the page's offset there (0 for an
 * absent page, as every directory has it).  The destination's 16-byte blocks are dealt out across the lanes (lane k writes blocks
 * k, k + 32, ...), each fed by aligned 8-byte source loads shifted into place, so one step of the warp loads and stores 512
 * consecutive bytes; the bytes before the first aligned block and after the last go one per lane.  Reads at most 7 bytes past a
 * page: inside the 1024 bytes that follow every data region and blob. */
__global__ void __launch_bounds__(APPEND_GATHER_THREADS) k_append_gather(const uint8_t *const *regions, const uint32_t *seg_region, const uint64_t *src_off,
                                                                         const uint32_t *len, uint64_t *dst_off, uint32_t n_segments, uint64_t n_pages, uint8_t *out) {
    const uint64_t page = ((uint64_t)blockIdx.x * APPEND_GATHER_THREADS + threadIdx.x) >> 5;
    const uint32_t lane = threadIdx.x & 31;
    if (page >= n_pages) return;
    const uint32_t l = len[page];
    if (l == 0) { if (lane == 0) dst_off[page] = 0; return; }
    const uint8_t *src = regions[seg_region[page % n_segments]] + src_off[page];
    uint8_t *dst = out + dst_off[page];
    const uint32_t head = min((uint32_t)((16 - ((uintptr_t)dst & 15)) & 15), l);
    const uint32_t n_blocks = (l - head) / 16, tail = head + n_blocks * 16;
    if (lane < head) dst[lane] = __ldg(src + lane);
    for (uint32_t k = lane; k < n_blocks; k += 32) {
        const uintptr_t sa = (uintptr_t)(src + head + 16 * k);
        const uint64_t *q = (const uint64_t *)(sa & ~(uintptr_t)7);
        const unsigned sh = (unsigned)(sa & 7) * 8;
        uint64_t a = __ldg(q), b = __ldg(q + 1);
        if (sh) { const uint64_t c = __ldg(q + 2); a = (a >> sh) | (b << (64 - sh)); b = (b >> sh) | (c << (64 - sh)); }
        *(uint4 *)(dst + head + 16 * k) = make_uint4((uint32_t)a, (uint32_t)(a >> 32), (uint32_t)b, (uint32_t)(b >> 32));
    }
    for (uint32_t i = tail + lane; i < l; i += 32) dst[i] = __ldg(src + i);
}

int gather_pages(const std::vector<const uint8_t *> &regions, const std::vector<uint32_t> &page_region, const std::vector<uint64_t> &src_off,
                 const std::vector<uint32_t> &len, const std::vector<uint64_t> &dst_off, uint8_t *out) {
    int rc;
    const uint64_t n = len.size();
    if (!n) return OG_OK;
    Scratch t;
    const uint8_t **d_regions; uint32_t *d_reg, *d_len; uint64_t *d_src, *d_dst;
    if ((rc = t.get(&d_regions, regions.size())) || (rc = t.get(&d_reg, n)) || (rc = t.get(&d_len, n)) || (rc = t.get(&d_src, n)) || (rc = t.get(&d_dst, n))) return rc;
    CU(cudaMemcpy(d_regions, regions.data(), regions.size() * sizeof(void *), cudaMemcpyHostToDevice));
    CU(cudaMemcpy(d_reg, page_region.data(), n * 4, cudaMemcpyHostToDevice));
    CU(cudaMemcpy(d_len, len.data(), n * 4, cudaMemcpyHostToDevice));
    CU(cudaMemcpy(d_src, src_off.data(), n * 8, cudaMemcpyHostToDevice));
    CU(cudaMemcpy(d_dst, dst_off.data(), n * 8, cudaMemcpyHostToDevice));
    k_append_gather<<<(unsigned)((n * 32 + APPEND_GATHER_THREADS - 1) / APPEND_GATHER_THREADS), APPEND_GATHER_THREADS>>>(
        d_regions, d_reg, d_src, d_len, d_dst, (uint32_t)n, n, out);
    CU(cudaGetLastError());
    CU(cudaDeviceSynchronize()); /* t goes back to the pool */
    return OG_OK;
}

/* per probed series of the shard: its last time, and the range [a, b) of its segments that a span [lo, hi] overlaps */
static __global__ void k_append_probe(const uint32_t *series_seg_begin, const int64_t *seg_tmin, const int64_t *seg_tmax, const uint32_t *series,
                                      const int64_t *lo, const int64_t *hi, uint32_t n, int64_t *last, uint32_t *a_out, uint32_t *b_out) {
    const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= n) return;
    const uint32_t g0 = series_seg_begin[series[k]], g1 = series_seg_begin[series[k] + 1];
    last[k] = g1 > g0 ? seg_tmax[g1 - 1] : INT64_MIN;
    uint32_t a = g0, e = g1; /* first segment with tmax >= lo (segments of a series are time-ordered) */
    while (a < e) { const uint32_t m = (a + e) / 2; if (seg_tmax[m] < lo[k]) a = m + 1; else e = m; }
    uint32_t b = a; e = g1;   /* first segment from a with tmin > hi */
    while (b < e) { const uint32_t m = (b + e) / 2; if (seg_tmin[m] <= hi[k]) b = m + 1; else e = m; }
    a_out[k] = a - g0; b_out[k] = b - g0;
}

int probe_series(const og_shard *s, const std::vector<uint32_t> &series, const int64_t *lo, const int64_t *hi, Probe &out) {
    int rc;
    const uint32_t n = (uint32_t)series.size();
    out.last.assign(n, INT64_MIN); out.a.clear(); out.b.clear();
    if (!n) return OG_OK;
    Scratch t;
    uint32_t *d_ser, *d_a, *d_b; int64_t *d_lo, *d_hi, *d_last;
    if ((rc = t.get(&d_ser, n)) || (rc = t.get(&d_lo, n)) || (rc = t.get(&d_hi, n)) || (rc = t.get(&d_last, n)) || (rc = t.get(&d_a, n)) || (rc = t.get(&d_b, n))) return rc;
    CU(cudaMemcpy(d_ser, series.data(), n * 4ull, cudaMemcpyHostToDevice));
    if (lo) {
        CU(cudaMemcpy(d_lo, lo, n * 8ull, cudaMemcpyHostToDevice));
        CU(cudaMemcpy(d_hi, hi, n * 8ull, cudaMemcpyHostToDevice));
    } else {
        CU(cudaMemset(d_lo, 0, n * 8ull)); CU(cudaMemset(d_hi, 0, n * 8ull));
    }
    k_append_probe<<<(n + 127) / 128, 128>>>(s->d_series_seg_begin, s->d_tmin, s->d_tmax, d_ser, d_lo, d_hi, n, d_last, d_a, d_b);
    CU(cudaGetLastError());
    CU(cudaMemcpy(out.last.data(), d_last, n * 8ull, cudaMemcpyDeviceToHost));
    if (lo) {
        out.a.resize(n); out.b.resize(n);
        CU(cudaMemcpy(out.a.data(), d_a, n * 4ull, cudaMemcpyDeviceToHost));
        CU(cudaMemcpy(out.b.data(), d_b, n * 4ull, cudaMemcpyDeviceToHost));
    }
    return OG_OK;
}

/* the derived totals of a spliced directory: rows, page bytes, time pages that are neither const-delta nor one-row, the largest
 * segment, the time range.  Reads only each time page's header. */
__global__ void k_append_stats(const uint8_t *data, const uint64_t *off, const uint32_t *len, const uint32_t *rows, const int64_t *tmin,
                               const int64_t *tmax, uint32_t n_segments, uint32_t n_columns, unsigned long long *tot, uint32_t *max_rows,
                               long long *range, int *err) {
    const uint32_t g = blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= n_segments) return;
    unsigned long long bytes = 0;
    for (uint32_t c = 0; c <= n_columns; c++) bytes += len[(size_t)c * n_segments + g];
    const size_t ti = (size_t)n_columns * n_segments + g;
    TimeDesc t;
    const int rc = parse_time_page(data + off[ti], len[ti], t);
    if (rc != D_OK) { if (atomicCAS(err, 0, rc) == 0) err[1] = (int)g; return; }
    atomicAdd(&tot[0], (unsigned long long)rows[g]);
    atomicAdd(&tot[1], bytes);
    if (t.kind != 0 && t.kind != 3) atomicAdd(&tot[2], 1ull);
    atomicMax(max_rows, rows[g]);
    atomicMin(&range[0], (long long)tmin[g]);
    atomicMax(&range[1], (long long)tmax[g]);
}

/* k_append_splice over `runs`, then, when a run reads another region than the files', every referenced page copied from `regions`
 * into one new buffer (+1024 zero bytes).  The directory arrays and the buffer are taken from `own`. */
int splice_and_gather(const SegSrc src[3], const std::vector<Run> &runs, uint32_t n_out, uint32_t n_columns,
                             const std::vector<const uint8_t *> &regions, Scratch &own, Spliced &out) {
    int rc;
    const uint64_t n_pages = (uint64_t)(n_columns + 1) * n_out;
    out.n = n_out; out.n_columns = n_columns;
    Scratch tmp;
    uint32_t *region; Run *d_runs;
    if ((rc = own.get(&out.off, n_pages)) || (rc = own.get(&out.len, n_pages)) || (rc = own.get(&out.rows, n_out)) ||
        (rc = own.get(&out.series, n_out)) || (rc = own.get(&out.tmin, n_out)) || (rc = own.get(&out.tmax, n_out)) ||
        (rc = tmp.get(&region, n_out)) || (rc = tmp.get(&d_runs, runs.size())))
        return rc;
    if (n_out) {
        CU(cudaMemcpy(d_runs, runs.data(), runs.size() * sizeof(Run), cudaMemcpyHostToDevice));
        SpliceP p;
        for (int k = 0; k < 3; k++) p.src[k] = src[k];
        p.runs = d_runs; p.n_runs = (uint32_t)runs.size(); p.n_out = n_out; p.n_columns = n_columns;
        p.off = out.off; p.len = out.len; p.rows = out.rows; p.series = out.series; p.region = region; p.tmin = out.tmin; p.tmax = out.tmax;
        k_append_splice<<<(n_out + 127) / 128, 128>>>(p);
    }
    /* every page already lies in the files' region at the offsets just spliced: keep that region rather than copy the pages */
    if (std::all_of(runs.begin(), runs.end(), [](const Run &r) { return r.kind == SRC_FILES; })) { CU(cudaGetLastError()); return OG_OK; }
    uint64_t *sizes, *dst_off; const uint8_t **d_regions;
    if ((rc = tmp.get(&sizes, n_pages + 1)) || (rc = tmp.get(&dst_off, n_pages + 1)) || (rc = tmp.get(&d_regions, regions.size()))) return rc;
    CU(cudaMemcpy(d_regions, regions.data(), regions.size() * sizeof(void *), cudaMemcpyHostToDevice));
    k_append_sizes<<<(unsigned)((n_pages + 1 + 255) / 256), 256>>>(out.len, n_pages, sizes);
    {
        size_t tb = 0; void *t = nullptr;
        CU(cub::DeviceScan::ExclusiveSum(nullptr, tb, sizes, dst_off, n_pages + 1));
        if ((rc = tmp.get((uint8_t **)&t, tb))) return rc;
        CU(cub::DeviceScan::ExclusiveSum(t, tb, sizes, dst_off, n_pages + 1));
    }
    CU(cudaGetLastError());
    CU(cudaMemcpy(&out.data_len, dst_off + n_pages, 8, cudaMemcpyDeviceToHost));
    if ((rc = own.get(&out.data, out.data_len + 1024))) return rc;
    CU(cudaMemset(out.data + out.data_len, 0, 1024));
    if (n_pages)
        k_append_gather<<<(unsigned)((n_pages * 32 + APPEND_GATHER_THREADS - 1) / APPEND_GATHER_THREADS), APPEND_GATHER_THREADS>>>(
            d_regions, region, out.off, out.len, dst_off, n_out, n_pages, out.data);
    CU(cudaGetLastError());
    CU(cudaMemcpy(out.off, dst_off, n_pages * 8, cudaMemcpyDeviceToDevice));
    CU(cudaDeviceSynchronize()); /* tmp goes back to the pool */
    return OG_OK;
}

/* ---------------------------------------------------------------- shared with compaction (span_pass.h) */

int batch_cap_rows(uint64_t per_row, uint64_t floor_rows, const char *env, uint64_t *cap) {
    size_t fr = 0, tot = 0;
    CU(dev_mem_info(&fr, &tot));
    *cap = std::max<uint64_t>(floor_rows, (uint64_t)(fr / 4) / per_row);
    if (const char *ov = getenv(env)) *cap = std::max<uint64_t>(1, strtoull(ov, nullptr, 10)); /* test hook */
    *cap = std::min<uint64_t>(*cap, 1ull << 30);
    return OG_OK;
}

int encode_columns(const std::vector<int32_t> &types, const int64_t *d_times, const std::vector<uint8_t *> &d_cols, const uint8_t *d_ok,
                   size_t out_rows, const uint32_t *d_rows, uint32_t n, uint32_t rps, uint8_t *blob, uint64_t cap, NewSegs &ns, uint64_t *used) {
    int rc;
    const uint32_t nc = (uint32_t)types.size(), ncol1 = nc + 1;
    Scratch t;
    uint64_t *d_off; uint32_t *d_len;
    if ((rc = t.get(&d_off, (size_t)ncol1 * n)) || (rc = t.get(&d_len, (size_t)ncol1 * n))) return rc;
    CU(cudaMemset(d_len, 0, (size_t)ncol1 * n * 4)); CU(cudaMemset(d_off, 0, (size_t)ncol1 * n * 8));
    ns.off.assign((size_t)ncol1 * n, 0); ns.len.assign((size_t)ncol1 * n, 0);
    for (uint32_t c = 0; c <= nc; c++) {
        const bool is_time = c == nc;
        if (!is_time && types[c] == OG_TYPE_STRING) continue;
        uint64_t tot = 0;
        rc = encode_pages(is_time ? OG_TYPE_INT : types[c], is_time ? 1 : 0, is_time ? (const void *)d_times : (const void *)d_cols[c],
                          is_time ? nullptr : d_ok + (size_t)c * out_rows, d_rows, n, rps, blob + *used, cap - *used,
                          d_off + (size_t)c * n, d_len + (size_t)c * n, &tot, true);
        if (rc) return rc;
        CU(cudaMemcpy(ns.off.data() + (size_t)c * n, d_off + (size_t)c * n, n * 8ull, cudaMemcpyDeviceToHost));
        CU(cudaMemcpy(ns.len.data() + (size_t)c * n, d_len + (size_t)c * n, n * 4ull, cudaMemcpyDeviceToHost));
        for (uint32_t g = 0; g < n; g++) ns.off[(size_t)c * n + g] += *used;
        *used += tot;
    }
    return OG_OK;
}

int keep_blob(const int64_t *d_tmin, const int64_t *d_tmax, std::vector<uint32_t> rows, const uint8_t *blob, uint64_t used, Scratch &blobs,
              NewSegs &ns) {
    int rc;
    ns.tmin.resize(ns.n); ns.tmax.resize(ns.n); ns.rows = std::move(rows);
    CU(cudaMemcpy(ns.tmin.data(), d_tmin, ns.n * 8ull, cudaMemcpyDeviceToHost));
    CU(cudaMemcpy(ns.tmax.data(), d_tmax, ns.n * 8ull, cudaMemcpyDeviceToHost));
    if ((rc = blobs.get(&ns.blob, used + 1024))) return rc;
    if (used) CU(cudaMemcpy(ns.blob, blob, used, cudaMemcpyDeviceToDevice));
    CU(cudaMemset(ns.blob + used, 0, 1024));
    ns.bytes = used;
    return OG_OK;
}

int string_refusal(unsigned long long sid, const std::string &column, const char *pass) {
    set_error("series sid %llu: string column \"%s\" has values in a span %s re-encodes (there is no device string encoder)", sid, column.c_str(), pass);
    return OG_E_UNSUPPORTED;
}

int decode_failure(int device_code, uint32_t seg, const char *where) {
    set_error("segment %u of the %s failed to decode (device code %d)", seg, where, device_code);
    return map_dev_err(device_code);
}

int batches_source(const std::vector<NewSegs> &batches, uint32_t nc, uint32_t first_region, std::vector<const uint8_t *> &regions,
                   Scratch &own, SegSrc &out, std::vector<uint32_t> &m_first) {
    int rc;
    m_first.assign(batches.size() + 1, 0);
    for (size_t b = 0; b < batches.size(); b++) m_first[b + 1] = m_first[b] + batches[b].n;
    const uint32_t NM = m_first[batches.size()];
    if (!NM) return OG_OK;
    std::vector<uint64_t> off((size_t)(nc + 1) * NM); std::vector<uint32_t> len((size_t)(nc + 1) * NM), rows(NM), reg(NM);
    std::vector<int64_t> tmin(NM), tmax(NM);
    for (size_t b = 0; b < batches.size(); b++) {
        const NewSegs &B = batches[b];
        regions.push_back(B.blob);
        for (uint32_t g = 0; g < B.n; g++) {
            const uint32_t m = m_first[b] + g;
            for (uint32_t c = 0; c <= nc; c++) { off[(size_t)c * NM + m] = B.off[(size_t)c * B.n + g]; len[(size_t)c * NM + m] = B.len[(size_t)c * B.n + g]; }
            rows[m] = B.rows[g]; reg[m] = first_region + (uint32_t)b; tmin[m] = B.tmin[g]; tmax[m] = B.tmax[g];
        }
    }
    uint64_t *d_off; uint32_t *d_len, *d_rows, *d_reg; int64_t *d_tmin, *d_tmax;
    if ((rc = own.get(&d_off, off.size())) || (rc = own.get(&d_len, len.size())) || (rc = own.get(&d_rows, NM)) || (rc = own.get(&d_reg, NM)) ||
        (rc = own.get(&d_tmin, NM)) || (rc = own.get(&d_tmax, NM)))
        return rc;
    CU(cudaMemcpy(d_off, off.data(), off.size() * 8, cudaMemcpyHostToDevice));
    CU(cudaMemcpy(d_len, len.data(), len.size() * 4, cudaMemcpyHostToDevice));
    CU(cudaMemcpy(d_rows, rows.data(), NM * 4ull, cudaMemcpyHostToDevice));
    CU(cudaMemcpy(d_reg, reg.data(), NM * 4ull, cudaMemcpyHostToDevice));
    CU(cudaMemcpy(d_tmin, tmin.data(), NM * 8ull, cudaMemcpyHostToDevice));
    CU(cudaMemcpy(d_tmax, tmax.data(), NM * 8ull, cudaMemcpyHostToDevice));
    out = SegSrc{d_off, d_len, d_rows, d_tmin, d_tmax, d_reg, 0, nullptr, NM, nc};
    return OG_OK;
}

int spliced_totals(const Spliced &sd, uint32_t nc, ShardState &out, const char *who) {
    int rc;
    Scratch t;
    unsigned long long *d_tot; uint32_t *d_max; long long *d_range; int *d_err;
    if ((rc = t.get(&d_tot, 3)) || (rc = t.get(&d_max, 1)) || (rc = t.get(&d_range, 2)) || (rc = t.get(&d_err, 2))) return rc;
    const long long r0[2] = {INT64_MAX, INT64_MIN};
    CU(cudaMemset(d_tot, 0, 24)); CU(cudaMemset(d_max, 0, 4)); CU(cudaMemset(d_err, 0, 8));
    CU(cudaMemcpy(d_range, r0, 16, cudaMemcpyHostToDevice));
    if (sd.n) k_append_stats<<<(sd.n + 127) / 128, 128>>>(sd.data, sd.off, sd.len, sd.rows, sd.tmin, sd.tmax, sd.n, nc, d_tot, d_max, d_range, d_err);
    CU(cudaGetLastError());
    unsigned long long tot[3]; long long range[2]; int err[2];
    CU(cudaMemcpy(tot, d_tot, 24, cudaMemcpyDeviceToHost));
    CU(cudaMemcpy(&out.max_seg_rows, d_max, 4, cudaMemcpyDeviceToHost));
    CU(cudaMemcpy(range, d_range, 16, cudaMemcpyDeviceToHost));
    CU(cudaMemcpy(err, d_err, 8, cudaMemcpyDeviceToHost));
    if (err[0]) { set_error("segment %d: time page failed to parse after %s (device code %d)", err[1], who, err[0]); return OG_E_CORRUPT; }
    out.n_rows = tot[0]; out.page_bytes = tot[1]; out.irregular_time_pages = tot[2]; out.tmin = range[0]; out.tmax = range[1];
    return OG_OK;
}

int install_state(og_shard *s, og_shard &out, Scratch &own, Spliced &sd, const std::vector<uint32_t> &series_seg_begin,
                  const std::vector<uint64_t> &sids, const std::vector<int32_t> &types, const std::vector<std::string> &names) {
    int rc;
    const size_t n_series = sids.size();
    out.device = s->device; out.n_series = (uint32_t)n_series; out.n_segments = sd.n; out.n_columns = sd.n_columns;
    out.sids = sids; out.col_types = types; out.col_names = names; out.h_series_seg_begin = series_seg_begin;
    if ((rc = dalloc(&out.d_series_seg_begin, n_series + 1)) || (rc = dalloc(&out.d_sids, n_series))) return rc;
    CU(cudaMemcpy(out.d_series_seg_begin, series_seg_begin.data(), (n_series + 1) * 4, cudaMemcpyHostToDevice));
    if (n_series) CU(cudaMemcpy(out.d_sids, sids.data(), n_series * 8, cudaMemcpyHostToDevice));
    auto take = [&](void *p) { own.bufs.erase(std::find(own.bufs.begin(), own.bufs.end(), p)); };
    for (void *p : {(void *)sd.off, (void *)sd.len, (void *)sd.rows, (void *)sd.series, (void *)sd.tmin, (void *)sd.tmax, (void *)sd.data}) take(p);
    out.d_page_off = sd.off; out.d_page_len = sd.len; out.d_seg_rows = sd.rows; out.d_seg_series = sd.series; out.d_tmin = sd.tmin; out.d_tmax = sd.tmax;
    out.d_data = sd.data; out.data_len = sd.data_len; out.owns_data = true;
    CU(cudaDeviceSynchronize());
    std::swap(static_cast<ShardState &>(*s), static_cast<ShardState &>(out));
    s->reset_il();
    return OG_OK;
}

/* ---------------------------------------------------------------- files into a shard */

/* the files join `s` (span_pass.h).  Everything from the probe on is one path for both producers of the new files. */
int add_files(og_shard *s, const og_shard_desc *files, const uint32_t *file_flags, uint32_t n_files, const char *who, DeviceFiles *dev) {
    int rc;
    /* ---- checks; schema union with the shard's columns (sorted by name), series union with its sids (ascending) ---- */
    const uint32_t onc = s->n_columns, ONSER = s->n_series, ONSEG = s->n_segments;
    std::map<std::string, int32_t> schema;
    for (uint32_t c = 0; c < onc; c++) schema[s->col_names[c]] = s->col_types[c];
    if (schema.size() != onc) { set_error("the shard holds two columns of one name"); return OG_E_UNSUPPORTED; }
    std::map<uint64_t, uint32_t> series_of_sid;
    if ((rc = scan_files(files, n_files, who, schema, series_of_sid))) return rc;
    std::map<uint64_t, uint32_t> old_of_sid;
    for (uint32_t i = 0; i < ONSER; i++) {
        if (!old_of_sid.emplace(s->sids[i], i).second) { set_error("the shard holds sid %llu twice", (unsigned long long)s->sids[i]); return OG_E_UNSUPPORTED; }
        series_of_sid[s->sids[i]] = 0;
    }
    std::vector<std::string> names; std::vector<int32_t> types;
    for (auto &kv : schema) { names.push_back(kv.first); types.push_back(kv.second); }
    std::vector<uint64_t> sids;
    for (auto &kv : series_of_sid) { kv.second = (uint32_t)sids.size(); sids.push_back(kv.first); }
    const uint32_t nc = (uint32_t)names.size(), NSER = (uint32_t)sids.size();
    std::vector<int32_t> col_of_old(nc, -1);
    for (uint32_t c = 0; c < onc; c++) col_of_old[std::lower_bound(names.begin(), names.end(), s->col_names[c]) - names.begin()] = (int32_t)c;
    std::vector<int64_t> old_of(NSER, -1);
    for (auto &kv : old_of_sid) old_of[series_of_sid[kv.first]] = kv.second;
    /* ---- the new files' directory; per series their ordered segments (file order) and out-of-order segments ---- */
    FileDir fd;
    if ((rc = build_file_dir(files, n_files, names, fd))) return rc;
    const uint32_t NN = fd.n;
    std::vector<std::vector<uint32_t>> ordered(NSER), ooo(NSER);
    og_merge_info info{}; info.n_files = n_files;
    if ((rc = split_segments(files, n_files, file_flags, fd, series_of_sid, sids, ordered, ooo, info))) return rc;
    /* ---- per series of the shard that takes new segments: its last time and the segments its span overlaps (device) ---- */
    std::vector<uint32_t> probe_u, probe_old; std::vector<int64_t> probe_lo, probe_hi;
    std::vector<int64_t> span_lo(NSER, INT64_MAX), span_hi(NSER, INT64_MIN);
    for (uint32_t u = 0; u < NSER; u++) {
        span_hull(ooo[u], fd, &span_lo[u], &span_hi[u]);
        if (old_of[u] >= 0 && (!ordered[u].empty() || !ooo[u].empty())) {
            probe_u.push_back(u); probe_old.push_back((uint32_t)old_of[u]); probe_lo.push_back(span_lo[u]); probe_hi.push_back(span_hi[u]);
        }
    }
    std::vector<uint32_t> old_a(NSER, 0), old_b(NSER, 0);
    Probe pr;
    if ((rc = probe_series(s, probe_old, probe_lo.data(), probe_hi.data(), pr))) return rc;
    for (size_t k = 0; k < probe_u.size(); k++) {
        const uint32_t u = probe_u[k];
        /* the flush rule: a series' new ordered rows start after the last time the shard holds for it */
        if (!ordered[u].empty() && fd.tmin[ordered[u][0]] <= pr.last[k]) {
            set_error("series sid %llu: ordered file %u starts at %lld, not after the shard's last time %lld; only out-of-order files may overlap the shard",
                      (unsigned long long)sids[u], fd.src_file[ordered[u][0]], (long long)fd.tmin[ordered[u][0]], (long long)pr.last[k]);
            return OG_E_UNSUPPORTED;
        }
        old_a[u] = pr.a[k]; old_b[u] = pr.b[k];
    }
    /* ---- layout: per series the shard's segments then its new ordered ones (one time-ordered list of n_old + n_new); a span
       rewrites the list's [before, after_begin) with the out-of-order segments ---- */
    auto n_old = [&](uint32_t u) { return old_of[u] < 0 ? 0u : s->h_series_seg_begin[old_of[u] + 1] - s->h_series_seg_begin[old_of[u]]; };
    auto g0_old = [&](uint32_t u) { return old_of[u] < 0 ? 0u : s->h_series_seg_begin[old_of[u]]; };
    std::vector<uint32_t> before(NSER), after_begin(NSER);
    std::vector<int> span_of(NSER, -1);
    std::vector<Span> span_store;
    for (uint32_t u = 0; u < NSER; u++) {
        const uint32_t no = n_old(u);
        const auto &o = ordered[u];
        if (ooo[u].empty()) { before[u] = after_begin[u] = no + (uint32_t)o.size(); continue; }
        uint32_t na, nb; /* the same bounds over the new ordered segments, which follow the shard's */
        span_bounds(o, fd, span_lo[u], span_hi[u], &na, &nb);
        before[u] = old_a[u] < no ? old_a[u] : no + na;
        after_begin[u] = old_b[u] < no ? old_b[u] : no + nb;
        Span sp; sp.series = u;
        span_of[u] = (int)span_store.size();
        span_store.push_back(std::move(sp));
    }
    /* ---- the new files on the device: uploaded, validated and transcoded, or taken over from the flush ---- */
    std::unique_ptr<og_shard> nw;
    std::vector<uint32_t> new_rows;
    if ((rc = dev ? place_files(files, n_files, names, types, s->device, fd, *dev, nw, new_rows)
                  : upload_files(files, n_files, names, types, s->device, fd, nw, new_rows)))
        return rc;
    s->reset_il(); /* the copies describe the old layout: their memory serves the pass */
    Scratch d_maps;
    int32_t *d_col_old;
    if ((rc = d_maps.get(&d_col_old, nc))) return rc;
    CU(cudaMemcpy(d_col_old, col_of_old.data(), nc * 4ull, cudaMemcpyHostToDevice));
    SegSrc src[3] = {};
    src[SRC_SHARD] = SegSrc{s->d_page_off, s->d_page_len, s->d_seg_rows, s->d_tmin, s->d_tmax, nullptr, 0, d_col_old, ONSEG, onc};
    src[SRC_FILES] = SegSrc{nw->d_page_off, nw->d_page_len, nw->d_seg_rows, nw->d_tmin, nw->d_tmax, nullptr, 1, nullptr, NN, nc};
    EventTimer timer;
    CU(timer.start());
    /* ---- merge: the spans' source segments spliced into one directory (the shard's rows first, then the new files in sequence,
       ordered before out-of-order), then merge_spans ---- */
    std::vector<NewSegs> batches;
    Scratch blobs, msrc_own;
    if (!span_store.empty()) {
        std::vector<Run> runs;
        uint32_t n_src = 0;
        for (auto &sp : span_store) {
            const uint32_t u = sp.series, no = n_old(u);
            const auto &o = ordered[u];
            const uint32_t ob = std::min(before[u], no), oe = std::min(after_begin[u], no);
            if (oe > ob) { /* the shard's rows: one "file", older than every new one */
                runs.push_back(Run{n_src, g0_old(u) + ob, 0, SRC_SHARD});
                for (uint32_t k = 0; k < oe - ob; k++) { sp.src.push_back(n_src + k); sp.src_file.push_back(n_files); }
                n_src += oe - ob;
            }
            std::vector<uint32_t> news;
            for (uint32_t k = std::max(before[u], no); k < after_begin[u]; k++) news.push_back(o[k - no]);
            news.insert(news.end(), ooo[u].begin(), ooo[u].end());
            sort_oldest_first(news, fd, file_flags);
            for (uint32_t g : news) {
                runs.push_back(Run{n_src, g, 0, SRC_FILES});
                sp.src.push_back(n_src++); sp.src_file.push_back(fd.src_file[g]);
            }
            info.series_merged++;
            info.segments_rewritten_in += sp.src.size();
        }
        for (uint32_t u = 0; u < NSER; u++) for (uint32_t g : ooo[u]) info.out_of_order_rows += new_rows[g];
        Spliced ms;
        if ((rc = splice_and_gather(src, runs, n_src, nc, {s->d_data, nw->d_data}, msrc_own, ms))) return rc;
        { /* the rows of every source segment, spliced with the rest of its directory: one copy */
            std::vector<uint32_t> rows(n_src);
            CU(cudaMemcpy(rows.data(), ms.rows, n_src * 4ull, cudaMemcpyDeviceToHost));
            for (auto &sp : span_store)
                for (uint32_t i : sp.src) { sp.src_rows.push_back(rows[i]); sp.rows += rows[i]; }
        }
        SrcDir dir;
        dir.data = ms.data ? ms.data : nw->d_data; dir.page_off = ms.off; dir.page_len = ms.len; dir.seg_rows = ms.rows; dir.n_segments = ms.n; dir.n_columns = nc;
        std::vector<Span *> sp;
        for (auto &x : span_store) sp.push_back(&x);
        uint64_t replaced = 0;
        if ((rc = merge_spans(dir, runs, types, names, sp, sids, n_files, batches, blobs, &replaced))) return rc;
        info.rows_replaced = replaced;
    }
    /* ---- the merged segments as one source directory, each batch's blob its own region ---- */
    std::vector<uint32_t> m_first;
    std::vector<const uint8_t *> regions = {s->d_data, nw->d_data};
    Scratch m_own;
    if ((rc = batches_source(batches, nc, 2, regions, m_own, src[SRC_MERGED], m_first))) return rc;
    /* ---- the new directory as runs: per series the shard's segments before its span, new ordered ones before it, the span's
       merged segments, then the rest of both ---- */
    std::vector<Run> runs;
    std::vector<uint32_t> o_ssb(NSER + 1, 0);
    uint32_t NOUT = 0;
    auto emit = [&](uint32_t u, uint32_t k0, uint32_t k1) { /* positions [k0, k1) of series u's time-ordered list */
        const uint32_t no = n_old(u);
        if (std::min(k1, no) > k0) { runs.push_back(Run{NOUT, g0_old(u) + k0, u, SRC_SHARD}); NOUT += std::min(k1, no) - k0; }
        for (uint32_t k = std::max(k0, no); k < k1; k++) runs.push_back(Run{NOUT++, ordered[u][k - no], u, SRC_FILES});
        info.segments_kept += k1 - k0;
    };
    for (uint32_t u = 0; u < NSER; u++) {
        o_ssb[u] = NOUT;
        const uint32_t total = n_old(u) + (uint32_t)ordered[u].size();
        emit(u, 0, before[u]);
        if (span_of[u] >= 0) {
            const Span &sp = span_store[span_of[u]];
            if (sp.n_new) { runs.push_back(Run{NOUT, m_first[sp.batch] + sp.first_new, u, SRC_MERGED}); NOUT += sp.n_new; }
            info.segments_rewritten_out += sp.n_new;
        }
        emit(u, after_begin[u], total);
    }
    o_ssb[NSER] = NOUT;
    /* ---- the new directory, and the live pages gathered into a new data region or left in the files' one ---- */
    std::unique_ptr<og_shard> out(new og_shard);
    Scratch out_own;
    Spliced sd;
    if ((rc = splice_and_gather(src, runs, NOUT, nc, regions, out_own, sd))) return rc;
    if (!sd.data) { sd.data = nw->d_data; sd.data_len = nw->data_len; nw->d_data = nullptr; out_own.bufs.push_back(sd.data); }
    CU(timer.stop());
    /* ---- derived state ---- */
    if ((rc = spliced_totals(sd, nc, *out, "the append"))) return rc;
    /* the Snappy counters hold while every transcoded page is in the shard: the first merge drops them */
    out->rows_merged = s->rows_merged || !batches.empty();
    if (!out->rows_merged) {
        out->snappy_pages = s->snappy_pages + nw->snappy_pages;
        out->snappy_bytes_in = s->snappy_bytes_in + nw->snappy_bytes_in; out->snappy_bytes_out = s->snappy_bytes_out + nw->snappy_bytes_out;
    }
    out->page_bytes = out->page_bytes - out->snappy_bytes_out + out->snappy_bytes_in;
    CU(timer.ms(&info.merge_ms));
    info.rows_after_merge = out->n_rows;
    out->merge = info;
    return install_state(s, *out, out_own, sd, o_ssb, sids, types, names);
}

/* ---------------------------------------------------------------- the entry points that rewrite a shard or open one */

int rewrite_shard(og_shard *s, const char *verb, const std::function<int()> &pass) {
    std::lock_guard<std::mutex> lock(s->live->mu); /* og_query_create waits until the rewrite is done */
    if (s->live->n) { set_error("%u queries on this shard are still open: destroy them before %s", s->live->n, verb); return OG_E_STATE; }
    CU(cudaSetDevice(s->device));
    return pass();
}

int open_empty(og_shard **out, const std::function<int(og_shard *)> &pass) {
    *out = nullptr;
    int rc = ensure_device(); if (rc) return rc;
    std::unique_ptr<og_shard> s(new og_shard);
    CU(cudaGetDevice(&s->device));
    s->h_series_seg_begin = {0};
    if ((rc = pass(s.get()))) return rc;
    *out = s.release();
    return OG_OK;
}

} // namespace ogpu

using namespace ogpu;

extern "C" {

OG_API int og_shard_open_files(const og_shard_desc *files, const uint32_t *file_flags, uint32_t n_files, og_shard **out) {
    if (!files || !out || n_files == 0) { set_error("null argument or no files"); return OG_E_INVAL; }
    return open_empty(out, [&](og_shard *s) { return add_files(s, files, file_flags, n_files, "og_shard_open_files", nullptr); });
}

OG_API int og_shard_append_files(og_shard *s, const og_shard_desc *files, const uint32_t *file_flags, uint32_t n_files) {
    if (!s || !files || n_files == 0) { set_error("null argument or no files"); return OG_E_INVAL; }
    return rewrite_shard(s, "appending files", [&] { return add_files(s, files, file_flags, n_files, "og_shard_append_files", nullptr); });
}

OG_API int og_shard_merge_info(const og_shard *s, og_merge_info *out) {
    if (!s || !out) { set_error("null argument"); return OG_E_INVAL; }
    *out = s->merge;
    return OG_OK;
}

} // extern "C"
