/*
 * fused_multi.cuh — K5, the general fused kernels: decode + filter + time-bucket + reduce, one thread per segment, NOTHING
 * materialised.  k_fused_multi serves the queries that touch several field columns and/or carry a WHERE on fields and that
 * k_fused_cols does not take (og_stats.path 4); k_fused_segment, its one-column form without a filter, serves single-column
 * queries over any codec, nulls or time codec (path 1, and the segments k_fused_il leaves over).
 *
 * The tile path writes every decoded column of a tile of segments to HBM (17 B per row and column, written and read back)
 * before it filters and reduces; here each column of the segment is a PULL iterator (ColIter, decode.cuh) and time comes from
 * a TimeIter, so a row's columns meet in registers: WHERE is evaluated on them (lib/binaryfilterfunc/functions.go:632
 * semantics: NULL never matches, ordered tests pass NaN), the surviving row is accumulated into the open window's partials,
 * and only window partials leave the thread (edges / per-series cells through SegWindows; k_window_reduce and k_fused_cols
 * write the same layout, so k_fix_edges and the merges are shared).  Pages are read front to back, and consecutive 8-byte
 * reads of one thread hit the sector/line its previous read brought into L1: DRAM traffic stays at the page bytes.
 *
 * Replaces (for <= OG_MULTI_MAXC columns): readSegmentRecord (tssp_file.go:369) + decodeColumnData (reader.go:674) for every
 * codec the device knows + FilterByTime (reader.go:754) + FilterByField (reader.go:895-974, functions.go:632)
 * + aggregateCursor (aggregate_cursor.go:306-356) + the per-window reducers (series_agg_func.gen.go:24-274).
 */
#pragma once
#include "agg_kernels.cuh"
#include <type_traits>

namespace ogpu {

/* Queries over more columns than this that k_fused_cols does not take run the materialise-tile path.  Building with
 * -DOG_WIDE_MULTI (tools/build_variants.sh wide:"-DOG_WIDE_MULTI") serves them here instead, with an exact instance for
 * each column count up to OG_MAX_COLS: the experiment behind the six-column row of DESIGN.md "Measured" (tools/bench_wide.py). */
#ifdef OG_WIDE_MULTI
#define OG_MULTI_MAXC OG_MAX_COLS
#else
#define OG_MULTI_MAXC 4
#endif

/* NCALL = number of calls (partials live in registers); SIMPLE = every call is count or sum (the shape configs[2] names): the
 * per-call switch of acc_row collapses to an add */
template <int NCOL, int NCALL, bool SIMPLE>
__global__ void __launch_bounds__(128) k_fused_multi(DirP d, QueryP q, ChunkP ch) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    const uint32_t seg = ch.seg_begin + i;
    if (seg >= ch.seg_end) return;
    const size_t e = 2 * (size_t)(seg - ch.seg_begin);
    const uint32_t rows = d.seg_rows[seg], series = d.seg_series[seg];
    auto no_rows = [&]() { ch.edge_bucket[e] = OG_NO_BUCKET; ch.edge_bucket[e + 1] = OG_NO_BUCKET; };
    if (d.seg_tmax[seg] < q.tmin || d.seg_tmin[seg] > q.tmax || rows == 0) { no_rows(); return; } /* segment pruning (location.go:276-280) */
    const size_t ti_idx = (size_t)d.n_columns * d.n_segments + seg;
    TimeDesc td;
    int rc = parse_time_page(d.data + d.page_off[ti_idx], d.page_len[ti_idx], td);
    if (rc != D_OK) { report_err(ch.err, rc, seg); no_rows(); return; }
    TimeIter ti; ti.init(td);
    ColIter col[NCOL];
#pragma unroll
    for (int k = 0; k < NCOL; k++) {
        const size_t pi = (size_t)q.col_index[k] * d.n_segments + seg;
        col[k].init(d.data + d.page_off[pi], d.page_len[pi], q.col_type[k], rows);
        if (col[k].err != D_OK) { report_err(ch.err, col[k].err, seg); no_rows(); return; }
    }
    Part parts[NCALL];
    SegWindows w(q, ch, seg, e, series);
    uint32_t r = 0;
    for (; r < rows; r++) {
        const int64_t t = ti.next();
        uint64_t v[NCOL]; bool ok[NCOL];
#pragma unroll
        for (int k = 0; k < NCOL; k++) { v[k] = 0; ok[k] = col[k].next(v[k]); } /* every column advances on every row, kept or not */
        if (t < q.tmin) continue;
        if (t > q.tmax) break;
        if (!w.enter(t, parts)) break;
        bool keep = true;
        if (q.n_filter == 1) { /* one compare term: no stack machine */
            const FilterP &f = q.filter[0];
            keep = false;
#pragma unroll
            for (int k = 0; k < NCOL; k++) if (f.col_slot == k) keep = ok[k] && term_pass(f, v[k]);
        } else if (q.n_filter) { /* RPN over compare terms; a NULL cell never matches (SURVEY App.B.12) */
            uint32_t stack = 0; int sp = 0;
            for (uint32_t fi = 0; fi < q.n_filter; fi++) {
                const FilterP &f = q.filter[fi];
                if (f.kind == OG_F_TERM) {
                    bool pass = false;
#pragma unroll
                    for (int k = 0; k < NCOL; k++) if (f.col_slot == k) pass = ok[k] && term_pass(f, v[k]);
                    stack |= (uint32_t)pass << sp; sp++;
                } else {
                    const uint32_t bb = (stack >> (sp - 1)) & 1, aa = (stack >> (sp - 2)) & 1;
                    const uint32_t rr = f.kind == OG_F_AND ? (aa & bb) : (aa | bb);
                    sp -= 2; stack &= ~(3u << sp); stack |= rr << sp; sp++;
                }
            }
            keep = stack & 1;
        }
        if (!keep) continue;
#pragma unroll
        for (int c = 0; c < NCALL; c++) {
            const CallP &cp = q.calls[c];
#pragma unroll
            for (int k = 0; k < NCOL; k++) {
                if (cp.col_slot != k || !ok[k]) continue;
                if (SIMPLE) { /* count: += 1; sum: sequential add in row order (integerSumReduce / floatSumReduce) */
                    if (cp.func == OG_AGG_COUNT) parts[c].v += 1;
                    else if (cp.type == OG_TYPE_FLOAT) parts[c].v = d2u(u2d(parts[c].v) + u2d(v[k]));
                    else parts[c].v += v[k];
                    parts[c].ok = 1;
                } else acc_row(cp.func, cp.type, parts[c], v[k], t);
            }
        }
    }
    if (r == rows) { /* the pages were walked to their last row (a scan that stops at tmax leaves the rest unread) */
        ti.finish();
#pragma unroll
        for (int k = 0; k < NCOL; k++) col[k].finish();
    }
    if (ti.err != D_OK) report_err(ch.err, ti.err, seg);
    for (int k = 0; k < NCOL; k++) if (col[k].err != D_OK) report_err(ch.err, col[k].err, seg);
    w.end(parts);
}

/* One column, no WHERE (og_stats.path 1, and the segments k_fused_il leaves over): the row loop of k_fused_multi without the
 * filter, run once per codec kind so that ColIter's codec switch folds away.  Sum, count, max over the int64 column of configs[2]
 * (H100 80GB HBM3, 400 W): this kernel 35.4 ms, k_fused_multi<1, 3, false> 48 ms, the push-decoder kernel it replaced 40.4 ms.  `list` (sorted segment
 * ids, `n` of them) selects the segments of the chunk that k_fused_il did not take, compacted so that warps stay full;
 * list == nullptr: every segment of the chunk. */
template <int NC>
__global__ void __launch_bounds__(128) k_fused_segment(DirP d, QueryP q, ChunkP ch, const uint32_t *list, uint32_t n) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint32_t seg = list ? list[i] : ch.seg_begin + i;
    const size_t e = 2 * (size_t)(seg - ch.seg_begin);
    const uint32_t rows = d.seg_rows[seg], series = d.seg_series[seg];
    auto no_rows = [&]() { ch.edge_bucket[e] = OG_NO_BUCKET; ch.edge_bucket[e + 1] = OG_NO_BUCKET; };
    if (d.seg_tmax[seg] < q.tmin || d.seg_tmin[seg] > q.tmax || rows == 0) { no_rows(); return; } /* segment pruning (location.go:276-280) */
    const size_t ti_idx = (size_t)d.n_columns * d.n_segments + seg;
    TimeDesc td;
    int rc = parse_time_page(d.data + d.page_off[ti_idx], d.page_len[ti_idx], td);
    if (rc != D_OK) { report_err(ch.err, rc, seg); no_rows(); return; }
    TimeIter ti; ti.init(td);
    ColIter col;
    const size_t pi = (size_t)q.col_index[0] * d.n_segments + seg;
    col.init(d.data + d.page_off[pi], d.page_len[pi], q.col_type[0], rows);
    if (col.err != D_OK) { report_err(ch.err, col.err, seg); no_rows(); return; }
    Part parts[NC];
    SegWindows w(q, ch, seg, e, series);
    uint32_t r = 0;
    auto walk = [&](auto kind) {
        col.kind = decltype(kind)::value; /* a constant from here on: value() reduces to this codec's case */
        for (; r < rows; r++) {
            const int64_t t = ti.next();
            uint64_t v = 0;
            const bool ok = col.next(v);
            if (t < q.tmin) continue;
            if (t > q.tmax) break;
            if (!w.enter(t, parts)) break;
            if (ok) {
#pragma unroll
                for (int c = 0; c < NC; c++) acc_row(q.calls[c].func, q.calls[c].type, parts[c], v, t);
            }
        }
    };
    using I = ColIter;
    switch (col.kind) {
    case I::K_ONE: walk(std::integral_constant<int, I::K_ONE>{}); break;
    case I::K_F_RAW: walk(std::integral_constant<int, I::K_F_RAW>{}); break;
    case I::K_F_GORILLA: walk(std::integral_constant<int, I::K_F_GORILLA>{}); break;
    case I::K_F_SAME: walk(std::integral_constant<int, I::K_F_SAME>{}); break;
    case I::K_F_RLE: walk(std::integral_constant<int, I::K_F_RLE>{}); break;
    case I::K_I_CONST: walk(std::integral_constant<int, I::K_I_CONST>{}); break;
    case I::K_I_S8B: walk(std::integral_constant<int, I::K_I_S8B>{}); break;
    case I::K_I_RAW: walk(std::integral_constant<int, I::K_I_RAW>{}); break;
    case I::K_B_BITS: walk(std::integral_constant<int, I::K_B_BITS>{}); break;
    default: walk(std::integral_constant<int, I::K_ABSENT>{}); break; /* an all-null page (string columns never run here) */
    }
    if (r == rows) { /* the pages were walked to their last row (a scan that stops at tmax leaves the rest unread) */
        ti.finish();
        col.finish();
    }
    if (ti.err != D_OK) report_err(ch.err, ti.err, seg);
    if (col.err != D_OK) report_err(ch.err, col.err, seg);
    w.end(parts);
}

} // namespace ogpu
