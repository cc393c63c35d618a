/*
 * flush.cu — rows into a shard (DESIGN.md (d) "Flushing rows into a shard"): og_shard_append_rows flushes a memtable snapshot into
 * an open shard, og_shard_open_rows into an empty one.  The reference sorts, splits and encodes every flushed series on host cores
 * (include/ogpu.h lists the code); here the rows go to the device once and the flush ends in the files' producer slot of add_files
 * (merge.cu), so the probe, spans, merge, splice, gather, stats and swap are the path og_shard_append_files runs.
 *
 *   host   check the description (fields against the shard's columns by name), the series in ascending sid, and per series its
 *          last time in the shard (k_append_probe).  Then per batch of series (rows under the merge's device-memory budget):
 *          times, bitmaps and dense values packed into one staging buffer, one host-to-device copy.  A series is charged its
 *          rows plus the 1000-row segment slots of its two parts, so many short series make small batches.
 *   device k_flush_expand   warp per chunk of 8192 rows of a (series, column), its first value counted on the host from the
 *                           bitmap: bitmap bits by ballot, dense value index by __popc of the lanes before,
 *                           values scattered into per-row cells and validity bytes ([column][row], as k_merge_decode writes them)
 *          StableSortPairs  by time inside each series (cub segmented sort): equal times keep arrival order
 *          k_flush_split    thread per series: the first sorted row after `last`.  A series' rows at or before it (out of order)
 *                           sort before the rest, so the two parts are two spans, (series, 0) and (series, 1), and no run of
 *                           equal times crosses them
 *          k_flush_row_span thread per sorted row: its span
 *          k_merge_heads, scan, k_merge_combine (span_pass.h): each column of a run of equal times takes its last non-null value in
 *                           arrival order (every row ranks as its own file), 1000-row segments from each span's first row, a flag
 *                           per (span, column) that holds a value
 *          encode_columns   the encoders of og_encode_pages into the batch's blob
 *   files  the ordered file holds every series' span 1, the out-of-order file every span 0; a column without a value in a span has
 *          no page there, a column without a value in a file is not one of its columns.  The live pages are gathered from the
 *          batch blobs into one region laid out as build_file_dir places a file set, which add_files takes over (DeviceFiles).
 *
 * The out-of-order file is decoded once more by the merge of add_files: those rows are few, and one merge path serves files and
 * rows (DESIGN.md (d) names merging them straight from the sorted rows as the next step).
 */
#include <algorithm>
#include <chrono>
#include <cstring>
#include <map>
#include <memory>
#include <string>
#include <vector>

#include "internal.h"
#include "span_pass.h"

namespace ogpu {

/* one (series, column) of a batch: its values at stage + val_off (8 bytes each, 1 for bool), its bitmap bits from bit bit0 of
 * stage + bm_off (no bitmap: every row valid) */
struct FlushTask { uint64_t val_off, bm_off; uint32_t row0, rows, col, bit0; };
constexpr uint64_t NO_BITMAP = ~0ull;
constexpr uint32_t FLUSH_CHUNK = 8192; /* rows of one expand task: a long series is spread over many warps */

__global__ void k_flush_expand(const uint8_t *stage, const FlushTask *tasks, uint32_t n_tasks, const int32_t *types, uint32_t R, uint64_t *cells,
                               uint8_t *ok) {
    const uint32_t w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (w >= n_tasks) return;
    const FlushTask tk = tasks[w];
    const bool is_bool = types[tk.col] == OG_TYPE_BOOL;
    const uint8_t *val = stage + tk.val_off, *bm = tk.bm_off == NO_BITMAP ? nullptr : stage + tk.bm_off;
    uint64_t *cv = cells + (size_t)tk.col * R + tk.row0;
    uint8_t *ov = ok + (size_t)tk.col * R + tk.row0;
    uint32_t dense = 0; /* non-null values before this step of 32 rows */
    for (uint32_t r0 = 0; r0 < tk.rows; r0 += 32) {
        const uint32_t r = r0 + lane;
        bool has = false;
        if (r < tk.rows) {
            const uint32_t b = tk.bit0 + r;
            has = bm ? ((bm[b >> 3] >> (b & 7)) & 1) != 0 : true;
        }
        const uint32_t m = __ballot_sync(0xffffffffu, has);
        if (r < tk.rows) {
            uint64_t v = 0;
            if (has) {
                const uint32_t d = dense + __popc(m & ((1u << lane) - 1));
                v = is_bool ? (uint64_t)val[d] : ((const uint64_t *)val)[d];
            }
            cv[r] = v; ov[r] = has ? 1 : 0;
        }
        dense += __popc(m);
    }
}

/* thread per series k of the batch (rows [row0[k], row0[k + 1]) sorted by time): span 2k holds its rows t <= last[k], span 2k + 1
 * the rest */
__global__ void k_flush_split(const int64_t *t, const uint32_t *row0, const int64_t *last, uint32_t n, uint32_t *span_row0) {
    const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= n) return;
    uint32_t a = row0[k], e = row0[k + 1];
    const int64_t L = last[k];
    span_row0[2 * k] = a;
    while (a < e) { const uint32_t m = (a + e) / 2; if (t[m] <= L) a = m + 1; else e = m; }
    span_row0[2 * k + 1] = a;
    if (k == n - 1) span_row0[2 * n] = row0[n];
}

/* thread per sorted row: the span that holds it (the last span starting at or before it: empty spans never hold a row) */
__global__ void k_flush_row_span(const uint32_t *span_row0, uint32_t n_spans, uint32_t R, uint32_t *row_span) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= R) return;
    uint32_t lo = 0, hi = n_spans;
    while (hi - lo > 1) { const uint32_t m = (lo + hi) / 2; if (span_row0[m] <= i) lo = m; else hi = m; }
    row_span[i] = lo;
}

static uint64_t value_width(int32_t type) { return type == OG_TYPE_BOOL ? 1 : 8; }

/* set bits of bm in [bit0, bit0 + n) */
static uint64_t count_bits(const uint8_t *bm, uint64_t bit0, uint64_t n) {
    uint64_t c = 0, b = bit0, e = bit0 + n;
    for (; b < e && (b & 7); b++) c += (bm[b >> 3] >> (b & 7)) & 1;
    for (; b + 64 <= e; b += 64) { uint64_t w; memcpy(&w, bm + (b >> 3), 8); c += (uint64_t)__builtin_popcountll(w); }
    for (; b < e; b++) c += (bm[b >> 3] >> (b & 7)) & 1;
    return c;
}

/* the host checks of og_rows_desc against the shard's columns; `order` gets the series with rows, ascending by sid */
static int check_rows(const og_shard *s, const og_rows_desc *d, std::vector<uint32_t> &order, uint64_t *rows_in) {
    if (d->flags) { set_error("og_rows_desc.flags must be 0 (got %u)", d->flags); return OG_E_INVAL; }
    if ((d->n_fields && !d->fields) || (d->n_series && !d->series)) { set_error("null fields or series"); return OG_E_INVAL; }
    if (d->n_fields > 64) { set_error("%u fields (limit 64)", d->n_fields); return OG_E_INVAL; }
    std::map<std::string, uint32_t> seen;
    for (uint32_t f = 0; f < d->n_fields; f++) {
        const std::string name = d->fields[f].name ? d->fields[f].name : "";
        const int32_t ty = d->fields[f].type;
        if (!seen.emplace(name, f).second) { set_error("field \"%s\" appears twice", name.c_str()); return OG_E_INVAL; }
        if (ty == OG_TYPE_STRING) { set_error("field \"%s\" is a string field: there is no device string encoder", name.c_str()); return OG_E_UNSUPPORTED; }
        if (ty != OG_TYPE_INT && ty != OG_TYPE_FLOAT && ty != OG_TYPE_BOOL) { set_error("field \"%s\": unknown type %d", name.c_str(), ty); return OG_E_INVAL; }
        for (uint32_t c = 0; c < s->n_columns; c++)
            if (s->col_names[c] == name && s->col_types[c] != ty) {
                set_error("column \"%s\" has type %d in the shard and %d in the rows", name.c_str(), s->col_types[c], ty); return OG_E_TYPE;
            }
    }
    std::map<uint64_t, uint32_t> sids;
    *rows_in = 0;
    for (uint32_t k = 0; k < d->n_series; k++) {
        const og_rows_series &sr = d->series[k];
        if (sr.sid == 0) { set_error("series %u: sid 0", k); return OG_E_INVAL; }
        if (!sids.emplace(sr.sid, k).second) { set_error("sid %llu appears twice", (unsigned long long)sr.sid); return OG_E_INVAL; }
        if (sr.rows && (!sr.times || (d->n_fields && !sr.cols))) { set_error("sid %llu: null times or columns", (unsigned long long)sr.sid); return OG_E_INVAL; }
        for (uint32_t f = 0; f < d->n_fields && sr.rows; f++) {
            const og_colval_view &cv = sr.cols[f];
            const char *name = d->fields[f].name ? d->fields[f].name : "";
            if (cv.len == 0) continue;
            if ((uint32_t)cv.len != sr.rows) { set_error("sid %llu field \"%s\": len %d is neither 0 nor rows (%u)", (unsigned long long)sr.sid, name, cv.len, sr.rows); return OG_E_INVAL; }
            if (cv.type != d->fields[f].type) { set_error("sid %llu field \"%s\": column type %d, field type %d", (unsigned long long)sr.sid, name, cv.type, d->fields[f].type); return OG_E_INVAL; }
            if (cv.nil_count < 0 || cv.nil_count > cv.len || cv.bitmap_offset < 0) { set_error("sid %llu field \"%s\": nil_count %d or bitmap_offset %d out of range", (unsigned long long)sr.sid, name, cv.nil_count, cv.bitmap_offset); return OG_E_INVAL; }
            const uint64_t n_val = (uint64_t)(cv.len - cv.nil_count);
            if (cv.val_bytes != n_val * value_width(cv.type) || (n_val && !cv.val)) {
                set_error("sid %llu field \"%s\": val_bytes %llu for %llu non-null values", (unsigned long long)sr.sid, name, (unsigned long long)cv.val_bytes, (unsigned long long)n_val);
                return OG_E_INVAL;
            }
            if (!cv.bitmap ? cv.nil_count != 0 : count_bits(cv.bitmap, (uint64_t)cv.bitmap_offset, (uint64_t)cv.len) != n_val) {
                set_error("sid %llu field \"%s\": nil_count %d disagrees with the bitmap", (unsigned long long)sr.sid, name, cv.nil_count);
                return OG_E_INVAL;
            }
        }
        *rows_in += sr.rows;
    }
    for (auto &kv : sids) if (d->series[kv.second].rows) order.push_back(kv.second);
    if (order.empty()) { set_error("no rows"); return OG_E_INVAL; }
    return OG_OK;
}

/* a span's place in the batches: its segments [first, first + n) of batch `batch`, and which columns hold a value in it */
struct SpanOut { uint32_t batch = 0, first = 0, n = 0; std::vector<uint8_t> has; };

/* sort, split and encode every series; spans[2k + p] of series order[k], p = 0 out of order, 1 ordered */
static int flush_batches(const og_shard *s, const og_rows_desc *d, const std::vector<uint32_t> &order, std::vector<NewSegs> &batches,
                         Scratch &blobs, std::vector<SpanOut> &spans, og_rows_info &info) {
    int rc;
    const uint32_t nf = d->n_fields, NSER = (uint32_t)order.size();
    std::vector<int32_t> types(nf);
    for (uint32_t f = 0; f < nf; f++) types[f] = d->fields[f].type;
    /* the last time the shard holds for each series (INT64_MIN for a sid it lacks) */
    std::vector<int64_t> last(NSER, INT64_MIN);
    {
        std::map<uint64_t, uint32_t> old_of_sid;
        for (uint32_t i = 0; i < s->n_series; i++) old_of_sid[s->sids[i]] = i;
        std::vector<uint32_t> pk, po;
        for (uint32_t k = 0; k < NSER; k++) {
            auto it = old_of_sid.find(d->series[order[k]].sid);
            if (it != old_of_sid.end()) { pk.push_back(k); po.push_back(it->second); }
        }
        Probe pr;
        if ((rc = probe_series(s, po, nullptr, nullptr, pr))) return rc;
        for (size_t j = 0; j < pk.size(); j++) last[pk[j]] = pr.last[j];
    }
    /* A batch's scratch follows its rows (staging, cells, sort) and its output slots (segment slots and encoder blob, per slot as
       much as span_row_bytes charges a row).  Every non-empty part takes whole 1000-row segments, so a series is charged its rows
       plus the slots of its two parts: a one-row series costs a whole segment, and many short series make small batches. */
    const uint64_t stage_per_row = 8 + 9ull * nf;
    uint64_t cap_rows;
    if ((rc = batch_cap_rows(span_row_bytes(nf) + stage_per_row, MERGE_RPS, "OGPU_MERGE_BATCH_ROWS", &cap_rows))) return rc;
    auto slots = [](uint64_t n) { return (n + MERGE_RPS - 1) / MERGE_RPS * MERGE_RPS; };
    std::vector<uint64_t> weight(NSER);
    for (uint32_t k = 0; k < NSER; k++) {
        const og_rows_series &sr = d->series[order[k]];
        uint64_t n_ooo = 0;
        for (uint32_t r = 0; r < sr.rows; r++) n_ooo += sr.times[r] <= last[k];
        weight[k] = sr.rows + slots(n_ooo) + slots(sr.rows - n_ooo);
    }
    unsigned long long *d_rep; MergeErr *d_err; int32_t *d_types;
    Scratch keep;
    if ((rc = keep.get(&d_rep, 1)) || (rc = keep.get(&d_err, 1)) || (rc = keep.get(&d_types, nf))) return rc;
    CU(cudaMemset(d_rep, 0, 8)); CU(cudaMemset(d_err, 0, sizeof(MergeErr)));
    CU(cudaMemcpy(d_types, types.data(), nf * 4ull, cudaMemcpyHostToDevice));
    spans.assign(2 * (size_t)NSER, SpanOut{});
    uint32_t k0 = 0;
    while (k0 < NSER) {
        auto t0 = std::chrono::steady_clock::now();
        uint32_t k1 = k0; uint64_t R64 = 0, W = 0;
        while (k1 < NSER && (k1 == k0 || W + weight[k1] <= cap_rows)) { W += weight[k1]; R64 += d->series[order[k1++]].rows; }
        if (R64 >= 0xffffffffull) { set_error("a batch of the flush holds %llu rows (limit 2^32 - 2)", (unsigned long long)R64); return OG_E_UNSUPPORTED; }
        const uint32_t R = (uint32_t)R64, nser = k1 - k0;
        /* ---- the staging buffer: times [R], series first rows [nser + 1], last times [nser], tasks, then bitmaps and values ---- */
        auto up8 = [](uint64_t x) { return (x + 7) & ~7ull; };
        std::vector<uint32_t> row0(nser + 1, 0);
        for (uint32_t k = 0; k < nser; k++) row0[k + 1] = row0[k] + d->series[order[k0 + k]].rows;
        uint64_t pos = 0;
        const uint64_t o_times = pos; pos += 8ull * R;
        const uint64_t o_row0 = pos; pos = up8(pos + 4ull * (nser + 1));
        const uint64_t o_last = pos; pos += 8ull * nser;
        /* per (series, column) with values: where its values and bitmap bytes are staged */
        struct ColStage { uint64_t val_off, bm_off; uint32_t k, f; };
        std::vector<ColStage> cols;
        size_t n_tasks = 0;
        for (uint32_t k = 0; k < nser; k++) {
            const og_rows_series &sr = d->series[order[k0 + k]];
            for (uint32_t f = 0; f < nf; f++)
                if (sr.cols[f].len) { cols.push_back(ColStage{0, NO_BITMAP, k, f}); n_tasks += (sr.rows + FLUSH_CHUNK - 1) / FLUSH_CHUNK; }
        }
        const uint64_t o_tasks = pos; pos += sizeof(FlushTask) * n_tasks;
        for (ColStage &c : cols) {
            const og_rows_series &sr = d->series[order[k0 + c.k]];
            const og_colval_view &cv = sr.cols[c.f];
            pos = up8(pos); c.val_off = pos; pos += cv.val_bytes;
            if (cv.bitmap && cv.nil_count) { c.bm_off = pos; pos += ((cv.bitmap_offset & 7) + sr.rows + 7) / 8; }
        }
        /* per chunk of FLUSH_CHUNK rows: one expand task, its first value after the values of the chunks before it */
        std::vector<FlushTask> tasks;
        tasks.reserve(n_tasks);
        for (const ColStage &c : cols) {
            const og_rows_series &sr = d->series[order[k0 + c.k]];
            const og_colval_view &cv = sr.cols[c.f];
            const uint64_t w = value_width(cv.type), bit0 = (uint64_t)(cv.bitmap_offset & 7);
            uint64_t dense = 0;
            for (uint32_t c0 = 0; c0 < sr.rows; c0 += FLUSH_CHUNK) {
                const uint32_t n = std::min(FLUSH_CHUNK, sr.rows - c0);
                FlushTask tk{c.val_off + dense * w, NO_BITMAP, row0[c.k] + c0, n, c.f, 0};
                if (c.bm_off != NO_BITMAP) {
                    tk.bm_off = c.bm_off + (bit0 + c0) / 8; tk.bit0 = (uint32_t)((bit0 + c0) & 7);
                    dense += count_bits(cv.bitmap, (uint64_t)cv.bitmap_offset + c0, n);
                } else dense += n;
                tasks.push_back(tk);
            }
        }
        /* not value-initialised: every byte the device reads is written below */
        const uint64_t stage_bytes = up8(pos);
        std::unique_ptr<uint8_t[]> stage(new uint8_t[stage_bytes]);
        for (uint32_t k = 0; k < nser; k++) {
            const og_rows_series &sr = d->series[order[k0 + k]];
            memcpy(stage.get() + o_times + 8ull * row0[k], sr.times, 8ull * sr.rows);
        }
        for (const ColStage &c : cols) {
            const og_rows_series &sr = d->series[order[k0 + c.k]];
            const og_colval_view &cv = sr.cols[c.f];
            if (cv.val_bytes) memcpy(stage.get() + c.val_off, cv.val, cv.val_bytes);
            if (c.bm_off != NO_BITMAP) memcpy(stage.get() + c.bm_off, cv.bitmap + cv.bitmap_offset / 8, ((cv.bitmap_offset & 7) + sr.rows + 7) / 8);
        }
        memcpy(stage.get() + o_row0, row0.data(), 4ull * (nser + 1));
        for (uint32_t k = 0; k < nser; k++) memcpy(stage.get() + o_last + 8ull * k, &last[k0 + k], 8);
        if (!tasks.empty()) memcpy(stage.get() + o_tasks, tasks.data(), sizeof(FlushTask) * tasks.size());
        Scratch b;
        uint8_t *d_stage; uint32_t *span_row0, *row_span, *perm_in, *perm; int64_t *times_sorted; uint64_t *cells; uint8_t *ok, *span_has;
        const uint32_t nsp = 2 * nser;
        if ((rc = b.get(&d_stage, stage_bytes)) || (rc = b.get(&span_row0, nsp + 1)) || (rc = b.get(&row_span, R)) || (rc = b.get(&perm_in, R)) ||
            (rc = b.get(&perm, R)) || (rc = b.get(&times_sorted, R)) || (rc = b.get(&cells, (size_t)nf * R)) || (rc = b.get(&ok, (size_t)nf * R)) ||
            (rc = b.get(&span_has, (size_t)nsp * nf)))
            return rc;
        CU(cudaMemcpy(d_stage, stage.get(), stage_bytes, cudaMemcpyHostToDevice));
        info.phase_ms[0] += ms_since(t0);
        t0 = std::chrono::steady_clock::now();
        /* ---- expand, sort by time inside each series, split into spans, runs of equal times ---- */
        const int64_t *times = (const int64_t *)(d_stage + o_times);
        const uint32_t *d_row0 = (const uint32_t *)(d_stage + o_row0);
        CU(cudaMemset(ok, 0, (size_t)nf * R));
        CU(cudaMemset(span_has, 0, (size_t)nsp * nf));
        if (!tasks.empty())
            k_flush_expand<<<(unsigned)((tasks.size() * 32 + 127) / 128), 128>>>(d_stage, (const FlushTask *)(d_stage + o_tasks), (uint32_t)tasks.size(),
                                                                                  d_types, R, cells, ok);
        if ((rc = sort_spans(times, times_sorted, perm_in, perm, R, nser, d_row0, b))) return rc;
        k_flush_split<<<(nser + 127) / 128, 128>>>(times_sorted, d_row0, (const int64_t *)(d_stage + o_last), nser, span_row0);
        k_flush_row_span<<<(R + 255) / 256, 256>>>(span_row0, nsp, R, row_span);
        /* every row is its own "file": perm_in (the identity) never repeats, so no run is refused */
        SortedRows sr{times_sorted, perm, row_span, span_row0, cells, ok, R, nsp};
        if ((rc = find_runs(sr, perm_in, b, d_err))) return rc;
        CU(cudaDeviceSynchronize());
        info.phase_ms[1] += ms_since(t0);
        t0 = std::chrono::steady_clock::now();
        /* ---- the row rule into segment slots, then the encoders ---- */
        NewSegs ns;
        std::vector<uint32_t> seg_first;
        if ((rc = combine_and_encode(sr, types, d_types, b, d_rep, span_has, blobs, ns, seg_first))) return rc;
        std::vector<uint8_t> has((size_t)nsp * nf);
        if (!has.empty()) CU(cudaMemcpy(has.data(), span_has, has.size(), cudaMemcpyDeviceToHost));
        for (uint32_t j = 0; j < nsp; j++) {
            SpanOut &o = spans[2 * (size_t)k0 + j];
            o.batch = (uint32_t)batches.size(); o.first = seg_first[j]; o.n = seg_first[j + 1] - seg_first[j];
            o.has.assign(has.begin() + (size_t)j * nf, has.begin() + (size_t)(j + 1) * nf);
            for (uint32_t g = o.first; g < o.first + o.n; g++) (j & 1 ? info.ordered_rows : info.out_of_order_rows) += ns.rows[g];
        }
        info.segments_written += ns.n;
        batches.push_back(std::move(ns));
        info.phase_ms[2] += ms_since(t0);
        k0 = k1;
    }
    unsigned long long rep = 0;
    CU(cudaMemcpy(&rep, d_rep, 8, cudaMemcpyDeviceToHost));
    info.rows_replaced = rep;
    return OG_OK;
}

/* the two files of the flush (ordered first, each only when it holds rows) as descriptions over one device region that holds their
 * live pages as build_file_dir places a file set */
struct FlushFiles {
    struct File { std::vector<uint64_t> sids; std::vector<uint32_t> ssb{0}; std::vector<int64_t> tmin, tmax;
                  std::vector<std::vector<uint64_t>> off; std::vector<std::vector<uint32_t>> len; std::vector<uint32_t> cols;
                  std::vector<og_column_desc> cdesc; uint64_t bytes = 0; bool ooo = false; };
    std::vector<File> files;
    std::vector<og_shard_desc> descs;
    std::vector<uint32_t> flags;
};

static int build_files(const og_rows_desc *d, const std::vector<uint32_t> &order, const std::vector<NewSegs> &batches,
                       const std::vector<SpanOut> &spans, FlushFiles &ff, DeviceFiles &df) {
    int rc;
    const uint32_t nf = d->n_fields, NSER = (uint32_t)order.size();
    std::vector<const uint8_t *> regions;
    for (const NewSegs &ns : batches) regions.push_back(ns.blob);
    std::vector<uint32_t> page_region, page_len; std::vector<uint64_t> src_off, dst_off;
    uint64_t pos = 0;
    for (int part : {1, 0}) {
        FlushFiles::File F;
        F.ooo = part == 0;
        std::vector<uint8_t> kept(nf, 0);
        for (uint32_t k = 0; k < NSER; k++)
            for (uint32_t f = 0; f < nf; f++) kept[f] |= spans[2 * (size_t)k + part].has[f];
        for (uint32_t f = 0; f < nf; f++) if (kept[f]) F.cols.push_back(f);
        const uint32_t fc = (uint32_t)F.cols.size();
        F.off.assign(fc + 1, {}); F.len.assign(fc + 1, {});
        const uint64_t base = (pos + 15) & ~15ull; /* build_file_dir's place for the file */
        uint64_t fpos = 0;
        for (uint32_t k = 0; k < NSER; k++) {
            const SpanOut &o = spans[2 * (size_t)k + part];
            if (!o.n) continue;
            const NewSegs &B = batches[o.batch];
            for (uint32_t g = o.first; g < o.first + o.n; g++) {
                for (uint32_t j = 0; j <= fc; j++) {
                    const bool time = j == fc;
                    const uint32_t c = time ? nf : F.cols[j];
                    const uint32_t l = time || o.has[c] ? B.len[(size_t)c * B.n + g] : 0;
                    F.off[j].push_back(l ? fpos : 0); F.len[j].push_back(l);
                    if (!l) continue;
                    page_region.push_back(o.batch); src_off.push_back(B.off[(size_t)c * B.n + g]); page_len.push_back(l); dst_off.push_back(base + fpos);
                    fpos += l;
                }
                F.tmin.push_back(B.tmin[g]); F.tmax.push_back(B.tmax[g]); df.rows.push_back(B.rows[g]);
            }
            F.sids.push_back(d->series[order[k]].sid);
            F.ssb.push_back((uint32_t)F.tmin.size());
        }
        if (F.sids.empty()) continue;
        F.bytes = fpos;
        pos = base + fpos;
        ff.files.push_back(std::move(F));
    }
    df.data_len = pos;
    if ((rc = dalloc(&df.data, pos + 1024))) return rc;
    CU(cudaMemset(df.data, 0, pos + 1024));
    if ((rc = gather_pages(regions, page_region, src_off, page_len, dst_off, df.data))) return rc;
    for (FlushFiles::File &F : ff.files) {
        const uint32_t fc = (uint32_t)F.cols.size();
        for (uint32_t j = 0; j < fc; j++) {
            const og_rows_field &fld = d->fields[F.cols[j]];
            F.cdesc.push_back(og_column_desc{fld.name ? fld.name : "", fld.type, F.off[j].data(), F.len[j].data()});
        }
        og_shard_desc sd{};
        sd.data = df.data; /* a device address: add_files takes the region over and never reads files[].data */
        sd.data_len = F.bytes; sd.n_series = (uint32_t)F.sids.size(); sd.sids = F.sids.data(); sd.series_seg_begin = F.ssb.data();
        sd.n_segments = (uint32_t)F.tmin.size(); sd.seg_tmin = F.tmin.data(); sd.seg_tmax = F.tmax.data();
        sd.n_columns = fc; sd.columns = F.cdesc.data(); sd.time_page_off = F.off[fc].data(); sd.time_page_len = F.len[fc].data();
        ff.descs.push_back(sd);
        ff.flags.push_back(F.ooo ? OG_FILE_OUT_OF_ORDER : 0);
    }
    return OG_OK;
}

/* the flush of `d` into `s`; the caller holds the shard's live-query lock */
static int flush_rows(og_shard *s, const og_rows_desc *d, og_rows_info *info_out, const char *who) {
    int rc;
    og_rows_info info{};
    std::vector<uint32_t> order;
    if ((rc = check_rows(s, d, order, &info.rows_in))) return rc;
    info.series_in = d->n_series;
    std::vector<NewSegs> batches;
    Scratch blobs;
    std::vector<SpanOut> spans;
    if ((rc = flush_batches(s, d, order, batches, blobs, spans, info))) return rc;
    auto t0 = std::chrono::steady_clock::now();
    FlushFiles ff;
    DeviceFiles df;
    if ((rc = build_files(d, order, batches, spans, ff, df))) return rc;
    CU(cudaDeviceSynchronize());
    info.phase_ms[2] += ms_since(t0);
    t0 = std::chrono::steady_clock::now();
    { Scratch drop; drop.bufs.swap(blobs.bufs); } /* the batch blobs were gathered: back to the pool before the merge */
    if ((rc = add_files(s, ff.descs.data(), ff.flags.data(), (uint32_t)ff.descs.size(), who, &df))) return rc;
    info.phase_ms[3] = ms_since(t0);
    if (info_out) *info_out = info;
    return OG_OK;
}

} // namespace ogpu

using namespace ogpu;

extern "C" {

OG_API int og_shard_append_rows(og_shard *s, const og_rows_desc *rows, og_rows_info *info) {
    if (!s || !rows) { set_error("null argument"); return OG_E_INVAL; }
    return rewrite_shard(s, "appending rows", [&] { return flush_rows(s, rows, info, "og_shard_append_rows"); });
}

OG_API int og_shard_open_rows(const og_rows_desc *rows, og_shard **out, og_rows_info *info) {
    if (!rows || !out) { set_error("null argument"); return OG_E_INVAL; }
    return open_empty(out, [&](og_shard *s) { return flush_rows(s, rows, info, "og_shard_open_rows"); });
}

} // extern "C"
