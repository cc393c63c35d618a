/*
 * compact.cu — og_shard_compact: every series of an open shard re-cut into full segments, as the reference's level compaction
 * writes them (DESIGN.md (d) "Compacting a shard").
 *
 * The reference merges a series' records across the files it compacts and writes them through MsBuilder.WriteRecord ->
 * WriteData (engine/immutable/compact.go:175-242, msbuilder.go:1151), which cuts them into segments of R rows from the start of
 * the series (GetMaxRowsPerSegment4TsStore, default 1000); every column of the chunk schema gets a page in every segment
 * (stream_compact.go:303 mergeSchema, 833-840 newNilCol).  Here the rows of one shard are already merged and in time order, so
 * a re-cut row's output slot is known from prefix sums of the segment row counts:
 *
 *   host   per series, from the directory alone (rows and page lengths per segment): the first segment that breaks the layout,
 *          or the first segment when a column has pages in only some segments; the rows from there on and their new segment
 *          count.  Segments before it end at multiples of R and keep their bytes.
 *   device per batch of spans (scratch ~ output row slots, under a device-memory budget):
 *          k_compact_decode   one thread per (source segment, column), the time column counted as one: ColIter / TimeIter
 *                             straight into the row's slot (segment base + local / R, local % R)
 *          k_compact_check    one thread per output slot: times strictly ascend inside a span, seg_tmin / seg_tmax
 *          encode_columns     the encoders of og_encode_pages, raw page for a float segment Gorilla refuses; string columns
 *                             (null in every re-cut row) get an all-null page from k_compact_null_pages
 *   finish the new directory from runs of the shard's kept segments and the new ones (splice_and_gather), the live pages gathered
 *          into a new data region, k_append_stats for the totals, and install_state swaps the new state in whole.
 */
#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>

#include "decode.cuh"
#include "internal.h"
#include "span_pass.h"

namespace ogpu {

#define COMPACT_RPS_DEFAULT 1000u /* lib/util/util.go:72 */

__device__ __forceinline__ bool compact_claim(MergeErr *e, int code) { return atomicCAS(&e->code, 0, code) == 0; }

/* one thread per (source segment, column), the time column last: the segment's rows of that column into their output slots.
 * Source j's row k goes to local row local0[j] + k of its span, i.e. slot (out0[j] + local / R) * R + local % R. */
__global__ void k_compact_decode(SrcDir d, const int32_t *col_types, uint32_t nsrc, const uint32_t *src_seg, const uint32_t *src_local0,
                                 const uint32_t *src_out0, const uint32_t *src_span, uint32_t R, int64_t *out_t, uint8_t *const *out_cells,
                                 uint8_t *out_ok, size_t out_rows, MergeErr *err) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (uint64_t)nsrc * (d.n_columns + 1)) return;
    const uint32_t c = (uint32_t)(i / nsrc), j = (uint32_t)(i % nsrc);
    const uint32_t seg = src_seg[j], rows = d.seg_rows[seg];
    size_t g = src_out0[j] + src_local0[j] / R;
    uint32_t slot = src_local0[j] % R;
    if (c == d.n_columns) {
        const size_t ti = (size_t)d.n_columns * d.n_segments + seg;
        TimeDesc t;
        int rc = parse_time_page(d.data + d.page_off[ti], d.page_len[ti], t);
        if (rc == D_OK && t.rows != rows) rc = D_CORRUPT;
        if (rc == D_OK) {
            TimeIter it; it.init(t);
            for (uint32_t k = 0; k < rows; k++) {
                out_t[g * R + slot] = it.next();
                if (++slot == R) { slot = 0; g++; }
            }
            it.finish(); rc = it.err;
        }
        if (rc != D_OK && compact_claim(err, rc)) err->seg = (int)seg;
        return;
    }
    const size_t pi = (size_t)c * d.n_segments + seg;
    ColIter ci;
    ci.init(d.data + d.page_off[pi], d.page_len[pi], col_types[c], rows);
    if (ci.err == D_OK && ci.kind == ColIter::K_NULLMAP) { /* a string value: there is no device string encoder */
        if (compact_claim(err, M_STRING)) { err->seg = (int)seg; err->col = (int)c; err->span = (int)src_span[j]; }
        return;
    }
    const bool narrow = col_types[c] == OG_TYPE_BOOL;
    uint8_t *cells = out_cells[c], *ok = out_ok + (size_t)c * out_rows;
    for (uint32_t k = 0; k < rows; k++) {
        uint64_t v = 0;
        const bool has = ci.next(v);
        const size_t dst = g * R + slot;
        ok[dst] = has ? 1 : 0;
        if (narrow) cells[dst] = has ? (uint8_t)v : 0;
        else ((uint64_t *)cells)[dst] = has ? v : 0;
        if (++slot == R) { slot = 0; g++; }
    }
    ci.finish();
    if (ci.err != D_OK && compact_claim(err, ci.err)) err->seg = (int)seg;
}

/* one thread per output slot: times strictly ascend inside a span (across its new segments too: every segment but a span's last
 * is full, so the row before slot 0 is the slot before it); the first and last time of every new segment */
__global__ void k_compact_check(const int64_t *out_t, const uint32_t *seg_rows, const uint32_t *seg_span, uint32_t n_segments, uint32_t R,
                                int64_t *seg_tmin, int64_t *seg_tmax, MergeErr *err) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (uint64_t)n_segments * R) return;
    const uint32_t g = (uint32_t)(i / R), slot = (uint32_t)(i % R), rows = seg_rows[g];
    if (slot >= rows) return;
    const int64_t t = out_t[i];
    if (slot == 0) seg_tmin[g] = t;
    if (slot == rows - 1) seg_tmax[g] = t;
    const bool has_prev = slot > 0 || (g > 0 && seg_span[g - 1] == seg_span[g]);
    if (has_prev && out_t[i - 1] >= t && compact_claim(err, M_REPEAT)) { err->span = (int)seg_span[g]; err->time = (long long)t; }
}

/* one all-null string page per new segment, 8 bytes apart: [34 + 10][u32 BE rows] (the header write_header gives a segment whose
 * rows are all null; lib/encoding: the type's "full" code + 10) */
__global__ void k_compact_null_pages(const uint32_t *seg_rows, uint32_t n_segments, uint8_t *out) {
    const uint32_t g = blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= n_segments) return;
    const uint32_t r = seg_rows[g];
    uint8_t *p = out + 8ull * g;
    p[0] = 44; p[1] = (uint8_t)(r >> 24); p[2] = (uint8_t)(r >> 16); p[3] = (uint8_t)(r >> 8); p[4] = (uint8_t)r;
    p[5] = p[6] = p[7] = 0;
}

/* a series re-cut from segment `first` on (shard segment index) */
struct CSpan {
    uint32_t series, first, end;    /* shard segments [first, end) */
    uint64_t rows = 0, mask = 0;    /* mask: the columns with a page in some segment of the series */
    uint32_t n_new = 0, batch = 0, first_new = 0;
};

/* bytes one encoded page of r rows can take: header, bitmap, one value per row, rounded to 8 (<= MERGE_PAGE_BOUND) */
static uint64_t page_bound(uint32_t r) { return std::min<uint64_t>(MERGE_PAGE_BOUND, (14ull + (r + 7) / 8 + 8ull * r + 16 + 7) & ~7ull); }

static int compact_spans(og_shard *s, uint32_t R, const std::vector<uint32_t> &rows, std::vector<CSpan> &spans, std::vector<NewSegs> &batches, Scratch &blobs) {
    int rc;
    const uint32_t nc = s->n_columns, ncol1 = nc + 1;
    /* scratch per output slot: time 8, per column 8 + 1, int compaction 8, encoder staging per segment, blob */
    const uint64_t per_slot = 8 + 9ull * nc + 8 + (MERGE_PAGE_BOUND + R - 1) / R + (ncol1 * page_bound(R) + 8 + R - 1) / R;
    uint64_t cap;
    if ((rc = batch_cap_rows(per_slot, R, "OGPU_COMPACT_BATCH_ROWS", &cap))) return rc;
    Scratch keep;
    MergeErr *d_err; int32_t *d_types;
    if ((rc = keep.get(&d_err, 1)) || (rc = keep.get(&d_types, nc))) return rc;
    CU(cudaMemcpy(d_types, s->col_types.data(), nc * 4ull, cudaMemcpyHostToDevice));
    CU(cudaMemset(d_err, 0, sizeof(MergeErr)));
    SrcDir dir{s->d_data, s->d_page_off, s->d_page_len, s->d_seg_rows, s->n_segments, nc};
    size_t a = 0;
    while (a < spans.size()) {
        size_t b = a; uint64_t slots = 0;
        while (b < spans.size() && (b == a || slots + (uint64_t)spans[b].n_new * R <= cap)) slots += (uint64_t)spans[b++].n_new * R;
        if (slots >= 0xffffffffull) { set_error("a re-cut span holds %llu row slots (limit 2^32 - 2)", (unsigned long long)slots); return OG_E_UNSUPPORTED; }
        const uint32_t nsp = (uint32_t)(b - a);
        /* host lists: source segments with their first local row and their span's first new segment; new segments' rows and span */
        std::vector<uint32_t> h_seg, h_local0, h_out0, h_span, h_rows, h_seg_span;
        NewSegs ns;
        for (uint32_t k = 0; k < nsp; k++) {
            CSpan &sp = spans[a + k];
            sp.batch = (uint32_t)batches.size(); sp.first_new = ns.n;
            uint32_t local = 0;
            for (uint32_t g = sp.first; g < sp.end; g++) {
                h_seg.push_back(g); h_local0.push_back(local); h_out0.push_back(ns.n); h_span.push_back(k);
                local += rows[g];
            }
            for (uint32_t g = 0; g < sp.n_new; g++) { h_rows.push_back((uint32_t)std::min<uint64_t>(R, sp.rows - (uint64_t)g * R)); h_seg_span.push_back(k); }
            ns.n += sp.n_new;
        }
        const uint32_t nsrc = (uint32_t)h_seg.size(), NS = ns.n;
        const size_t out_rows = (size_t)NS * R;
        Scratch t;
        uint32_t *d_seg, *d_local0, *d_out0, *d_span, *d_rows, *d_seg_span; int64_t *out_t, *d_tmin, *d_tmax; uint8_t *out_ok; uint8_t **d_cols;
        std::vector<uint8_t *> h_cols(nc);
        if ((rc = t.get(&d_seg, nsrc)) || (rc = t.get(&d_local0, nsrc)) || (rc = t.get(&d_out0, nsrc)) || (rc = t.get(&d_span, nsrc)) ||
            (rc = t.get(&d_rows, NS)) || (rc = t.get(&d_seg_span, NS)) || (rc = t.get(&out_t, out_rows)) || (rc = t.get(&d_tmin, NS)) ||
            (rc = t.get(&d_tmax, NS)) || (rc = t.get(&out_ok, std::max<size_t>(1, (size_t)nc * out_rows))) || (rc = t.get(&d_cols, nc)))
            return rc;
        for (uint32_t c = 0; c < nc; c++)
            if ((rc = t.get(&h_cols[c], out_rows * (s->col_types[c] == OG_TYPE_BOOL ? 1 : 8)))) return rc;
        CU(cudaMemcpy(d_seg, h_seg.data(), nsrc * 4ull, cudaMemcpyHostToDevice));
        CU(cudaMemcpy(d_local0, h_local0.data(), nsrc * 4ull, cudaMemcpyHostToDevice));
        CU(cudaMemcpy(d_out0, h_out0.data(), nsrc * 4ull, cudaMemcpyHostToDevice));
        CU(cudaMemcpy(d_span, h_span.data(), nsrc * 4ull, cudaMemcpyHostToDevice));
        CU(cudaMemcpy(d_rows, h_rows.data(), NS * 4ull, cudaMemcpyHostToDevice));
        CU(cudaMemcpy(d_seg_span, h_seg_span.data(), NS * 4ull, cudaMemcpyHostToDevice));
        CU(cudaMemcpy(d_cols, h_cols.data(), nc * sizeof(uint8_t *), cudaMemcpyHostToDevice));
        const uint64_t nthr = (uint64_t)nsrc * ncol1;
        k_compact_decode<<<(unsigned)((nthr + 127) / 128), 128>>>(dir, d_types, nsrc, d_seg, d_local0, d_out0, d_span, R, out_t, d_cols, out_ok, out_rows, d_err);
        k_compact_check<<<(unsigned)((out_rows + 255) / 256), 256>>>(out_t, d_rows, d_seg_span, NS, R, d_tmin, d_tmax, d_err);
        CU(cudaGetLastError());
        MergeErr he;
        CU(cudaMemcpy(&he, d_err, sizeof he, cudaMemcpyDeviceToHost));
        if (he.code) {
            if (he.code == M_STRING) return string_refusal((unsigned long long)s->sids[spans[a + he.span].series], s->col_names[he.col], "compaction");
            if (he.code == M_REPEAT) {
                set_error("series sid %llu: time %lld does not follow the row before it inside a span compaction re-cuts (times must strictly ascend)",
                          (unsigned long long)s->sids[spans[a + he.span].series], he.time);
                return OG_E_CORRUPT;
            }
            return decode_failure(he.code, (uint32_t)he.seg, "shard");
        }
        /* encode; string columns of the series get an all-null page, columns a series lacks get none */
        uint8_t *blob;
        const uint64_t bcap = (uint64_t)NS * ncol1 * page_bound(R) + 8ull * NS;
        if ((rc = t.get(&blob, bcap))) return rc;
        uint64_t used = 0;
        if ((rc = encode_columns(s->col_types, out_t, h_cols, out_ok, out_rows, d_rows, NS, R, blob, bcap, ns, &used))) return rc;
        const bool any_string = std::any_of(s->col_types.begin(), s->col_types.end(), [](int32_t ty) { return ty == OG_TYPE_STRING; });
        const uint64_t nulls = used;
        if (any_string) {
            k_compact_null_pages<<<(NS + 127) / 128, 128>>>(d_rows, NS, blob + nulls);
            CU(cudaGetLastError());
            used += 8ull * NS;
        }
        for (uint32_t k = 0; k < nsp; k++) {
            const CSpan &sp = spans[a + k];
            for (uint32_t c = 0; c < nc; c++)
                for (uint32_t g = sp.first_new; g < sp.first_new + sp.n_new; g++) {
                    const size_t pi = (size_t)c * NS + g;
                    if (!((sp.mask >> c) & 1)) { ns.off[pi] = 0; ns.len[pi] = 0; }
                    else if (s->col_types[c] == OG_TYPE_STRING) { ns.off[pi] = nulls + 8ull * g; ns.len[pi] = 5; }
                }
        }
        if ((rc = keep_blob(d_tmin, d_tmax, std::move(h_rows), blob, used, blobs, ns))) return rc;
        batches.push_back(std::move(ns));
        a = b;
    }
    return OG_OK;
}

static int compact(og_shard *s, uint32_t R, og_compact_info &info) {
    int rc;
    const uint32_t nc = s->n_columns, NSER = s->n_series, NSEG = s->n_segments;
    /* ---- the plan, from the directory: per segment its rows and which columns have a page ---- */
    std::vector<uint32_t> len((size_t)(nc + 1) * NSEG), rows(NSEG);
    if (NSEG) {
        CU(cudaMemcpy(rows.data(), s->d_seg_rows, NSEG * 4ull, cudaMemcpyDeviceToHost));
        CU(cudaMemcpy(len.data(), s->d_page_len, len.size() * 4, cudaMemcpyDeviceToHost));
    }
    std::vector<CSpan> spans;
    for (uint32_t u = 0; u < NSER; u++) {
        const uint32_t g0 = s->h_series_seg_begin[u], g1 = s->h_series_seg_begin[u + 1];
        if (g1 == g0) continue;
        uint64_t any = 0, all = ~0ull >> (64 - std::max(nc, 1u));
        if (nc == 0) all = 0;
        for (uint32_t g = g0; g < g1; g++) {
            uint64_t m = 0;
            for (uint32_t c = 0; c < nc; c++) if (len[(size_t)c * NSEG + g]) m |= 1ull << c;
            any |= m; all &= m;
        }
        uint32_t k = g1;
        if (any != all) k = g0; /* a column in only some segments: the whole series */
        else
            for (uint32_t g = g0; g < g1; g++)
                if (rows[g] > R || (g + 1 < g1 && rows[g] < R)) { k = g; break; }
        if (k == g1) continue;
        CSpan sp; sp.series = u; sp.first = k; sp.end = g1; sp.mask = any;
        for (uint32_t g = k; g < g1; g++) sp.rows += rows[g];
        sp.n_new = (uint32_t)((sp.rows + R - 1) / R);
        spans.push_back(sp);
    }
    if (spans.empty()) return OG_OK; /* already compact: nothing is copied */
    s->reset_il(); /* the copies describe the old layout: their memory serves the pass */
    EventTimer timer;
    CU(timer.start());
    std::vector<NewSegs> batches;
    Scratch blobs;
    if ((rc = compact_spans(s, R, rows, spans, batches, blobs))) return rc;
    /* ---- the new segments as one source, the shard's own as another ---- */
    SegSrc src[3] = {};
    src[SRC_SHARD] = SegSrc{s->d_page_off, s->d_page_len, s->d_seg_rows, s->d_tmin, s->d_tmax, nullptr, 0, nullptr, NSEG, nc};
    std::vector<const uint8_t *> regions = {s->d_data, nullptr}; /* region 1 (files) is not used here */
    std::vector<uint32_t> m_first;
    Scratch m_own;
    if ((rc = batches_source(batches, nc, 2, regions, m_own, src[SRC_MERGED], m_first))) return rc;
    /* ---- the new directory as runs: per series its kept segments, then its new ones ---- */
    std::vector<Run> runs;
    std::vector<uint32_t> o_ssb(NSER + 1, 0);
    uint32_t NOUT = 0;
    size_t si = 0;
    for (uint32_t u = 0; u < NSER; u++) {
        o_ssb[u] = NOUT;
        const uint32_t g0 = s->h_series_seg_begin[u], g1 = s->h_series_seg_begin[u + 1];
        const CSpan *sp = si < spans.size() && spans[si].series == u ? &spans[si++] : nullptr;
        const uint32_t kept_end = sp ? sp->first : g1;
        if (kept_end > g0) { runs.push_back(Run{NOUT, g0, u, SRC_SHARD}); NOUT += kept_end - g0; info.segments_kept += kept_end - g0; }
        if (sp) {
            runs.push_back(Run{NOUT, m_first[sp->batch] + sp->first_new, u, SRC_MERGED}); NOUT += sp->n_new;
            info.series_rewritten++; info.segments_rewritten_in += sp->end - sp->first; info.segments_rewritten_out += sp->n_new;
            info.rows_rewritten += sp->rows;
        }
    }
    o_ssb[NSER] = NOUT;
    std::unique_ptr<og_shard> out(new og_shard);
    Scratch out_own;
    Spliced sd;
    if ((rc = splice_and_gather(src, runs, NOUT, nc, regions, out_own, sd))) return rc;
    CU(timer.stop());
    if ((rc = spliced_totals(sd, nc, *out, "compaction"))) return rc;
    /* the Snappy counters hold while every transcoded page is in the shard: a re-cut drops them, as a merge does */
    out->rows_merged = true;
    out->merge = s->merge;
    CU(timer.ms(&info.compact_ms));
    return install_state(s, *out, out_own, sd, o_ssb, s->sids, s->col_types, s->col_names);
}

} // namespace ogpu

using namespace ogpu;

extern "C" {

OG_API int og_shard_compact(og_shard *s, const og_compact_desc *d, og_compact_info *info) {
    if (!s || !d) { set_error("null argument"); return OG_E_INVAL; }
    if (d->flags) { set_error("og_compact_desc.flags must be 0 (got %u)", d->flags); return OG_E_INVAL; }
    if (d->rows_per_segment > 1000) { set_error("rows_per_segment must be 0 (1000) or 1..1000 (got %u)", d->rows_per_segment); return OG_E_INVAL; }
    const uint32_t R = d->rows_per_segment ? d->rows_per_segment : COMPACT_RPS_DEFAULT;
    return rewrite_shard(s, "compacting it", [&] {
        og_compact_info ci{};
        const int rc = compact(s, R, ci);
        if (rc == OG_OK && info) *info = ci;
        return rc;
    });
}

} // extern "C"
