/*
 * agg_kernels.cuh — the scan/aggregate kernels.
 *
 * Data flow of one query over one chunk of series (all arrays in HBM):
 *
 *   pages ──k_fused_segment──┐                       (thread per segment: decode + window partials, nothing materialised)
 *   pages ──k_decode_tile──> tile ──k_filter_tile──> keep ──k_window_reduce──┤   (generic path: any column mix, WHERE filters)
 *                                                                            v
 *                         interior windows -> cells[series][bucket]   first/last window of a segment -> edges[2*seg]
 *                                                                            │
 *                         k_fix_edges: ordered stitch of windows that span segments (prevBuf/currBuf, series_agg_reducer.gen.go:228-266)
 *                                                                            v
 *                         k_merge_groups: per (group, bucket) sequential fold over the group's series in shard order
 *                                         (AggTagSetCursor.RecordInit agg_tagset_cursor.go:1069) -> dense interval record
 */
#pragma once
#include "agg_ops.cuh"
#include "decode.cuh"
#include "internal.h"

namespace ogpu {

#define OG_NO_BUCKET 0xFFFFFFFFu

struct DirP { /* device directory */
    const uint8_t *data;
    const uint64_t *page_off; /* [(n_columns+1)*n_segments] */
    const uint32_t *page_len;
    const uint32_t *seg_series, *seg_rows, *series_seg_begin;
    const int64_t *seg_tmin, *seg_tmax;
    uint32_t n_segments, n_columns;
};

struct ChunkP { /* one chunk of whole series */
    uint32_t series_begin, series_end; /* global series range */
    uint32_t seg_begin, seg_end;       /* global segment range (contiguous) */
    Tri cells[OG_MAX_CALLS];           /* per-series window partials [ cell_idx(ch, series, b) ]: series-major (the layout of the
                                          per-series dense record), so a lane that walks its segment appends to one row whatever
                                          series its neighbours hold, and a thread-per-bucket merge reads consecutive addresses */
    uint32_t nb;                       /* buckets per series row (= QueryP.n_buckets) */
    Tri edges[OG_MAX_CALLS];           /* [ 2 * (seg - seg_begin) + {0 head, 1 tail} ] */
    uint32_t *edge_bucket;             /* [ 2 * (seg - seg_begin) ] OG_NO_BUCKET = absent */
    Tri gcells[OG_MAX_CALLS];          /* folded window partials [ b * gc_cols + col ] (one tagset, regular shard): col < gc_tail0 is a
                                          lane group of the fused kernel (32 series folded in-warp: interior and head windows),
                                          gc_tail0 + col the tail windows of that lane group, col >= gc_edge0 a block of 32
                                          consecutive series whose stitched edge windows k_fix_edges_fold folded (three blocks of
                                          columns: runs led by a head window of even / odd segment index, runs led by a tail
                                          window).  nullptr when unused */
    uint32_t gc_cols, gc_tail0, gc_edge0, gc_col0;
    uint32_t J;                        /* segments per series on a regular shard, else 0 */
    int *err;                          /* [0] first error code, [1] segment */
    int *flags;                        /* [0] != 0: some kernel wrote per-series cells in this run (the cell merges have work);
                                          [1] != 0: k_fused_il, k_fused_segment or k_fused_multi wrote edge windows
                                          (k_fix_edges_fold has work) */
};

__device__ __forceinline__ size_t cell_idx(const ChunkP &ch, uint32_t series, uint32_t b) { return (size_t)(series - ch.series_begin) * ch.nb + b; }

__device__ __forceinline__ void report_err(int *err, int code, uint32_t seg) {
    if (atomicCAS(&err[0], 0, code) == 0) err[1] = (int)seg;
}

__device__ __forceinline__ void store_part(const Tri &a, size_t i, const Part &p) {
    a.val[i] = p.v; a.ok[i] = (uint8_t)p.ok;
    if (a.tim) a.tim[i] = p.t;
}
__device__ __forceinline__ Part load_part(const Tri &a, size_t i) {
    Part p; p.ok = a.ok[i]; p.v = a.val[i]; p.t = a.tim ? a.tim[i] : 0; return p;
}
/* a per-series window partial; marks the cell matrix as in use */
__device__ __forceinline__ void store_cell(const ChunkP &ch, int call, uint32_t series, uint32_t b, const Part &p) {
    store_part(ch.cells[call], cell_idx(ch, series, b), p);
    ch.flags[0] = 1;
}

/* Where one segment's window partials go, for the kernels that walk a segment's rows in time order in one thread (k_fused_multi,
 * k_fused_segment): the first window with in-range rows (head) to edges[e], the last one (tail) to edges[e + 1], the windows
 * between to the per-series cells; edge_bucket names the head and tail buckets for k_fix_edges.  The caller accumulates the rows
 * of the open window into `parts` left to right, which keeps float sums in the reference's order (series_agg_func.gen.go:48-60).
 * The kernels keep their prologue (pruning, time page, edge_bucket of a segment without rows) inline: as a member of this struct
 * it changed the register allocation of several k_fused_multi instances. */
struct SegWindows {
    const QueryP &q; const ChunkP &ch;
    const uint32_t seg; const size_t e; const uint32_t series;
    uint32_t cur_b = OG_NO_BUCKET, head_b = OG_NO_BUCKET; bool head_done = false;
    int64_t we = 0; /* end of the open window */

    __device__ __forceinline__ SegWindows(const QueryP &q_, const ChunkP &ch_, uint32_t seg_, size_t e_, uint32_t series_)
        : q(q_), ch(ch_), seg(seg_), e(e_), series(series_) {}
    template <int NC> __device__ __forceinline__ void flush(const Part (&parts)[NC], bool final) {
        if (cur_b == OG_NO_BUCKET) return;
#pragma unroll
        for (int c = 0; c < NC; c++) {
            if (!head_done) store_part(ch.edges[c], e, parts[c]);
            else if (final) store_part(ch.edges[c], e + 1, parts[c]);
            else if (parts[c].ok) store_cell(ch, c, series, cur_b, parts[c]);
        }
        if (!head_done) { head_done = true; head_b = cur_b; }
    }
    /* an in-range row at time t: when t leaves the open window, that window is flushed and the partials start empty.
     * false: t lies past the query's buckets (cannot happen on a validated shard), the walk ends */
    template <int NC> __device__ __forceinline__ bool enter(int64_t t, Part (&parts)[NC]) {
        if (cur_b != OG_NO_BUCKET && t < we) return true;
        flush(parts, false);
        cur_b = bucket_of(t, q.start, q.interval);
        if (cur_b >= q.n_buckets) { report_err(ch.err, D_CORRUPT, seg); cur_b = OG_NO_BUCKET; return false; }
        we = q.start + (int64_t)(cur_b + 1) * q.interval;
#pragma unroll
        for (int c = 0; c < NC; c++) parts[c] = part_empty();
        return true;
    }
    /* after the row loop: the open window is the tail (or the head, when it is the only one) */
    template <int NC> __device__ __forceinline__ void end(const Part (&parts)[NC]) {
        const uint32_t last_b = cur_b;
        const bool single = !head_done;
        flush(parts, true);
        ch.edge_bucket[e] = head_b;
        ch.edge_bucket[e + 1] = (single || head_b == OG_NO_BUCKET) ? OG_NO_BUCKET : last_b;
        if (head_b != OG_NO_BUCKET) ch.flags[1] = 1; /* edge windows written: k_fix_edges_fold has work */
    }
};

/* ------------------------------------------------------------------------------------------------------------
 * shard open: row counts, codec support and framing validation (one thread per segment)
 * ------------------------------------------------------------------------------------------------------------ */
__global__ void k_validate(DirP d, const int32_t *col_types, uint32_t *seg_rows, unsigned long long *totals /*[0]=rows [1]=page bytes [2]=time pages that are not const-delta / one-row*/,
                           uint32_t *max_rows, int *err) {
    uint32_t seg = blockIdx.x * blockDim.x + threadIdx.x;
    if (seg >= d.n_segments) return;
    size_t ti = (size_t)d.n_columns * d.n_segments + seg;
    TimeDesc t;
    int rc = parse_time_page(d.data + d.page_off[ti], d.page_len[ti], t);
    if (rc == D_OK && t.rows == 0) rc = D_CORRUPT;
    if (rc == D_OK) { /* the directory's time range must cover the page's times: bucket indices are derived from it and never re-checked */
        int64_t last = t.t0; bool unsorted = false; /* times must ascend (segments hold time-ordered rows, lib/record/record.go sort order) */
        if (t.kind == 0) last = (int64_t)((uint64_t)t.t0 + (uint64_t)(t.rows - 1) * t.delta); /* const-delta: closed form */
        else {
            TimeIter it; it.init(t);
            for (uint32_t i = 0; i < t.rows; i++) { const int64_t x = it.next(); unsorted |= x < last; last = x; }
            it.finish(); rc = it.err;
        }
        if (rc == D_OK && (t.t0 < d.seg_tmin[seg] || last > d.seg_tmax[seg] || last < t.t0 || unsorted)) rc = D_CORRUPT;
    }
    if (rc != D_OK) { report_err(err, rc, seg); seg_rows[seg] = 0; return; }
    seg_rows[seg] = t.rows;
    unsigned long long bytes = d.page_len[ti];
    for (uint32_t c = 0; c < d.n_columns; c++) {
        size_t pi = (size_t)c * d.n_segments + seg;
        uint32_t len = d.page_len[pi];
        if (len == 0) continue;
        bytes += len;
        PageHdr h;
        rc = parse_field_header(d.data + d.page_off[pi], len, col_types[c], t.rows, h);
        if (rc == D_OK && h.rows != t.rows) rc = D_CORRUPT;
        /* the decoders take one value per valid row: the bitmap must mark exactly the header's value count */
        if (rc == D_OK && h.bitmap && hdr_valid_rows(h) != h.rows - h.nil_count) rc = D_CORRUPT;
        if (rc == D_OK && !h.one_row && h.nil_count < h.rows) {
            if (h.block_len < 1) rc = D_CORRUPT;
            else {
                int tag = __ldg(h.block) >> 4, ty = col_types[c];
                if (ty == OG_TYPE_FLOAT) rc = (tag == 0 || tag == 3 || tag == 4 || tag == 5) ? D_OK : (tag == 1 || tag == 2 || tag == 6) ? D_UNSUPPORTED : D_CORRUPT;
                else if (ty == OG_TYPE_INT) rc = (tag == 1 || tag == 2 || tag == 4) ? D_OK : tag == 3 ? D_UNSUPPORTED : D_CORRUPT;
                else if (ty == OG_TYPE_BOOL) rc = tag == 1 ? D_OK : D_CORRUPT;
                else if (ty == OG_TYPE_STRING) rc = D_OK; /* only the header (row count, null bitmap) of a string page is ever read: count() */
                else rc = D_UNSUPPORTED;
            }
        }
        if (rc != D_OK) { report_err(err, rc, seg); return; }
    }
    atomicAdd(&totals[0], (unsigned long long)t.rows);
    atomicAdd(&totals[1], bytes);
    atomicMax(max_rows, t.rows);
    if (t.kind != 0 && t.kind != 3) atomicAdd(&totals[2], 1ull);
}

__global__ void k_fill_seg_series(const uint32_t *series_seg_begin, uint32_t n_series, uint32_t *seg_series) {
    uint32_t s = blockIdx.x;
    if (s >= n_series) return;
    for (uint32_t g = series_seg_begin[s] + threadIdx.x; g < series_seg_begin[s + 1]; g += blockDim.x) seg_series[g] = s;
}

/* ------------------------------------------------------------------------------------------------------------
 * generic path, step 1: materialise a tile of segments (thread per page; grid.y = column slot, last slot = time)
 *   vals[slot][(seg-tile_begin)*R + row]  expanded to one cell per row, okb = validity byte per row
 * ------------------------------------------------------------------------------------------------------------ */
struct TileP {
    uint32_t tile_begin, tile_end, R; /* R = rows reserved per segment */
    uint32_t S;                       /* segments per row of the tile (tile size rounded up to 32): cell (segment sl, row r)
                                         lives at r*S + sl, so threads that own consecutive segments and walk their rows in
                                         step read and write consecutive addresses */
    uint64_t *vals[OG_MAX_COLS];
    uint8_t *okb[OG_MAX_COLS];
    int64_t *times;
    uint8_t *keep;
};

__global__ void k_decode_tile(DirP d, QueryP q, TileP tp, int *err) {
    uint32_t seg = tp.tile_begin + blockIdx.x * blockDim.x + threadIdx.x;
    if (seg >= tp.tile_end) return;
    uint32_t slot = blockIdx.y;
    const size_t base = seg - tp.tile_begin, S = tp.S;
    uint32_t rows = d.seg_rows[seg];
    if (slot == q.n_cols) {
        size_t ti = (size_t)d.n_columns * d.n_segments + seg;
        TimeDesc t;
        int rc = parse_time_page(d.data + d.page_off[ti], d.page_len[ti], t);
        if (rc == D_OK) {
            TimeIter it; it.init(t);
            for (uint32_t i = 0; i < t.rows; i++) tp.times[base + i * S] = it.next();
            it.finish(); rc = it.err;
        }
        if (rc != D_OK) report_err(err, rc, seg);
        return;
    }
    size_t pi = (size_t)q.col_index[slot] * d.n_segments + seg;
    uint64_t *out = tp.vals[slot] + base; uint8_t *okb = tp.okb[slot] + base;
    ColIter it;
    it.init(d.data + d.page_off[pi], d.page_len[pi], q.col_type[slot], rows);
    for (uint32_t i = 0; i < rows; i++) { uint64_t v = 0; okb[i * S] = it.next(v); out[i * S] = v; } /* null rows: 0, validity 0 */
    it.finish();
    if (it.err != D_OK) report_err(err, it.err, seg);
}

/* step 2: row mask = inside [tmin,tmax] AND WHERE RPN (one thread per row; SURVEY App.B.12 semantics) */
__device__ __forceinline__ bool term_pass(const FilterP &f, uint64_t raw) {
    if (f.type == OG_TYPE_FLOAT || (f.type == OG_TYPE_INT && f.const_is_float)) {
        double v = f.type == OG_TYPE_FLOAT ? u2d(raw) : (double)(int64_t)raw;
        double c = f.const_is_float ? f.fval : (double)f.ival;
        switch (f.op) {
        case OG_OP_LT: return !(v >= c);
        case OG_OP_LTE: return !(v > c);
        case OG_OP_GT: return !(v <= c);
        case OG_OP_GTE: return !(v < c);
        case OG_OP_EQ: return !(v != c);
        default: return !(v == c);
        }
    }
    int64_t v = f.type == OG_TYPE_BOOL ? (int64_t)(raw != 0) : (int64_t)raw, c = f.ival;
    switch (f.op) {
    case OG_OP_LT: return !(v >= c);
    case OG_OP_LTE: return !(v > c);
    case OG_OP_GT: return !(v <= c);
    case OG_OP_GTE: return !(v < c);
    case OG_OP_EQ: return !(v != c);
    default: return !(v == c);
    }
}

__global__ void k_filter_tile(DirP d, QueryP q, TileP tp) {
    size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    size_t total = (size_t)tp.S * tp.R;
    if (idx >= total) return;
    uint32_t row = (uint32_t)(idx / tp.S), sl = (uint32_t)(idx % tp.S);
    if (sl >= tp.tile_end - tp.tile_begin) return;
    if (row >= d.seg_rows[tp.tile_begin + sl]) { tp.keep[idx] = 0; return; }
    int64_t t = tp.times[idx];
    bool keep = t >= q.tmin && t <= q.tmax;
    if (keep && q.n_filter) {
        uint32_t stack = 0; int sp = 0;
        for (uint32_t i = 0; i < q.n_filter; i++) {
            const FilterP &f = q.filter[i];
            if (f.kind == OG_F_TERM) {
                bool pass = tp.okb[f.col_slot][idx] && term_pass(f, tp.vals[f.col_slot][idx]);
                stack |= (uint32_t)pass << sp; sp++;
            } else {
                uint32_t b = (stack >> (sp - 1)) & 1, a = (stack >> (sp - 2)) & 1;
                uint32_t r = f.kind == OG_F_AND ? (a & b) : (a | b);
                sp -= 2; stack &= ~(3u << sp); stack |= r << sp; sp++;
            }
        }
        keep = stack & 1;
    }
    tp.keep[idx] = keep;
}

/* step 3: one thread per segment walks its rows in time order (threads of a warp own consecutive segments and move row by row
 * together, so every load is coalesced in the r*S + sl layout); the rows of a window are accumulated left to right, which keeps
 * float sums in the reference's order (series_agg_func.gen.go:48-60).  Windows are those of the rows inside [tmin, tmax]; rows
 * removed by the WHERE mask do not contribute, a window whose rows were all removed yields an invalid partial. */
__global__ void k_window_reduce(DirP d, QueryP q, TileP tp, ChunkP ch) {
    uint32_t sl = blockIdx.x * blockDim.x + threadIdx.x;
    uint32_t seg = tp.tile_begin + sl;
    if (seg >= tp.tile_end) return;
    const uint32_t rows = d.seg_rows[seg], series = d.seg_series[seg];
    const size_t S = tp.S, e = 2 * (size_t)(seg - ch.seg_begin);
    Part parts[OG_MAX_CALLS];
    uint32_t cur_b = OG_NO_BUCKET, head_b = OG_NO_BUCKET; bool head_done = false;
    int64_t we = 0;
    auto flush = [&](bool final) {
        if (cur_b == OG_NO_BUCKET) return;
        for (uint32_t c = 0; c < q.n_calls; c++) {
            if (!head_done) store_part(ch.edges[c], e, parts[c]);
            else if (final) store_part(ch.edges[c], e + 1, parts[c]);
            else if (parts[c].ok) store_cell(ch, (int)c, series, cur_b, parts[c]);
        }
        if (!head_done) { head_done = true; head_b = cur_b; }
    };
    for (uint32_t r = 0; r < rows; r++) {
        const size_t ix = (size_t)r * S + sl;
        const int64_t t = tp.times[ix];
        if (t < q.tmin) continue;
        if (t > q.tmax) break;
        if (cur_b == OG_NO_BUCKET || t >= we) {
            flush(false);
            cur_b = bucket_of(t, q.start, q.interval);
            if (cur_b >= q.n_buckets) { report_err(ch.err, D_CORRUPT, seg); cur_b = OG_NO_BUCKET; break; } /* cannot happen on a validated shard */
            we = q.start + (int64_t)(cur_b + 1) * q.interval;
#pragma unroll
            for (uint32_t c = 0; c < OG_MAX_CALLS; c++) parts[c] = part_empty();
        }
        if (!tp.keep[ix]) continue;
#pragma unroll
        for (uint32_t c = 0; c < OG_MAX_CALLS; c++) {
            if (c >= q.n_calls) break;
            const CallP &cp = q.calls[c];
            if (tp.okb[cp.col_slot][ix]) acc_row(cp.func, cp.type, parts[c], tp.vals[cp.col_slot][ix], t);
        }
    }
    flush(true);
    ch.edge_bucket[e] = head_b;
    ch.edge_bucket[e + 1] = (head_b == OG_NO_BUCKET || cur_b == head_b) ? OG_NO_BUCKET : cur_b;
}

/* ------------------------------------------------------------------------------------------------------------
 * ordered stitch of windows that span segment boundaries (prevBuf/currBuf, series_agg_reducer.gen.go:228-266)
 * ------------------------------------------------------------------------------------------------------------ */
struct EdgeRuns { uint32_t hb, tb, s_end; bool head_leader; };
/* the (up to two) windows of `seg` that may continue in neighbouring segments: its head window leads a run unless the previous
 * segment's last window is the same bucket; its tail window always leads */
__device__ __forceinline__ EdgeRuns edge_runs(const DirP &d, const ChunkP &ch, uint32_t seg, uint32_t series) {
    EdgeRuns r;
    const uint32_t s_first = d.series_seg_begin[series];
    r.s_end = d.series_seg_begin[series + 1];
    const uint32_t *eb = ch.edge_bucket;
    const size_t e = 2 * (size_t)(seg - ch.seg_begin);
    r.hb = eb[e]; r.tb = eb[e + 1];
    r.head_leader = true;
    if (r.hb != OG_NO_BUCKET && seg > s_first) { /* previous edge = tail(seg-1) if present else head(seg-1) */
        const size_t pe = e - 2;
        const uint32_t pb = eb[pe + 1] != OG_NO_BUCKET ? eb[pe + 1] : eb[pe];
        if (pb != OG_NO_BUCKET && pb == r.hb) r.head_leader = false;
    }
    return r;
}
/* partial of the run led by edge `which` of `seg` for one call: ordered left-to-right merge of the edges of that bucket */
__device__ __forceinline__ Part edge_stitch(const QueryP &q, const ChunkP &ch, const EdgeRuns &r, uint32_t seg, int which, uint32_t c) {
    const CallP &cp = q.calls[c];
    const uint32_t *eb = ch.edge_bucket;
    const size_t e = 2 * (size_t)(seg - ch.seg_begin);
    const uint32_t b = which == 0 ? r.hb : r.tb;
    Part acc = load_part(ch.edges[c], e + which);
    if (which == 1 || r.tb == OG_NO_BUCKET) { /* the run continues into later segments only from the last edge of this segment */
        for (uint32_t nx = seg + 1; nx < r.s_end; nx++) {
            const size_t ne = 2 * (size_t)(nx - ch.seg_begin);
            if (eb[ne] != b) break; /* includes OG_NO_BUCKET */
            acc = series_merge(cp.func, cp.type, acc, load_part(ch.edges[c], ne));
            if (eb[ne + 1] != OG_NO_BUCKET) break; /* that segment has a distinct tail window: run ends at its head */
        }
    }
    return acc;
}

/* thread per segment: stitched windows go to the per-series cells */
__global__ void k_fix_edges(DirP d, QueryP q, ChunkP ch) {
    uint32_t seg = ch.seg_begin + blockIdx.x * blockDim.x + threadIdx.x;
    if (seg >= ch.seg_end) return;
    const uint32_t series = d.seg_series[seg];
    const EdgeRuns r = edge_runs(d, ch, seg, series);
    if (r.hb == OG_NO_BUCKET) return; /* no in-range rows */
    for (int which = 0; which < 2; which++) {
        if (which == 0 && !r.head_leader) continue;
        if (which == 1 && r.tb == OG_NO_BUCKET) continue;
        const uint32_t b = which == 0 ? r.hb : r.tb;
        if (b >= q.n_buckets) { report_err(ch.err, D_CORRUPT, seg); continue; } /* a directory time range that lies about its page */
        for (uint32_t c = 0; c < q.n_calls; c++) {
            const Part acc = edge_stitch(q, ch, r, seg, which, c);
            if (acc.ok) store_cell(ch, (int)c, series, b, acc);
        }
    }
}

__device__ __forceinline__ Part shfl_xor_part(const Part &p, int o, bool with_time) {
    Part r; r.v = __shfl_xor_sync(0xffffffffu, p.v, o); r.ok = __shfl_xor_sync(0xffffffffu, p.ok, o);
    r.t = with_time ? __shfl_xor_sync(0xffffffffu, p.t, o) : 0;
    return r;
}
/* butterfly fold of 32 partials with the tagset update rules: group_update is commutative for count/sum and symmetric in its
 * selector tie-breaks (equal value -> earlier time; equal time -> larger value), so every lane ends with the same cell */
__device__ __forceinline__ Part warp_fold(int func, int type, bool multi, Part p, bool with_time) {
#pragma unroll
    for (int o = 16; o; o >>= 1) { const Part other = shfl_xor_part(p, o, with_time); group_update(func, type, multi, p, other); }
    return p;
}
__device__ __forceinline__ bool call_has_time(const QueryP &q, uint32_t c) { return q.calls[c].func >= OG_AGG_MIN && !(q.multi && q.calls[c].func <= OG_AGG_MAX); }
__device__ __forceinline__ int call_ftype(const QueryP &q, uint32_t c) { return q.calls[c].func == OG_AGG_COUNT ? OG_TYPE_INT : q.calls[c].type; }

/* regular shards, one tagset: warp per (block of 32 consecutive series, segment index); the lanes' stitched windows of one
 * bucket are folded in-warp into ONE cell of the folded matrix (a column of the block).  Blocks whose series do not agree
 * on the bucket (irregular time grids) fall back to per-series cells.  Segments whose edge windows k_fused_il folded in the warp
 * have no edge_bucket entries; when no kernel of this chunk wrote an edge window the launch returns at once. */
__global__ void k_fix_edges_fold(DirP d, QueryP q, ChunkP ch) {
    if (ch.flags[1] == 0) return;
    const uint32_t w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    const uint32_t n_blk = (ch.series_end - ch.series_begin + 31) / 32;
    if (w >= n_blk * ch.J) return;
    const uint32_t blk = w / ch.J, j = w % ch.J;
    const uint32_t series = ch.series_begin + blk * 32 + lane;
    const bool in = series < ch.series_end;
    const uint32_t seg = in ? d.series_seg_begin[series] + j : 0;
    EdgeRuns r; r.hb = r.tb = OG_NO_BUCKET; r.head_leader = false; r.s_end = 0;
    if (in) r = edge_runs(d, ch, seg, series);
    /* Every warp of a block stores with plain stores, so two warps of one block (two segment indices) must never write the
     * same (bucket, column).  Once some segments fold their edges in k_fused_il, the run of a bucket X may be led by different
     * segment indices in different series of the block: by tail(j) in a series whose segment j is stitched, by head(j+1) in
     * one whose segment j was folded; and by head(j) in a series whose segment j starts in X (a range that cuts segment j,
     * a coarser cadence) next to head(j+1) in one whose segment j was folded with its tail in X.  Hence three columns per
     * block: runs led by a tail window, and runs led by a head window of even and of odd j.  That suffices on the shards
     * the plan folds (segment index j covers one [seg_tmin, seg_tmax] in every series): tails of one bucket all come from
     * one j (times ascend with j), and heads from at most j and j+1 — if a series had a head-led run at X from j and another
     * one from j+2, segment j+1 would lie wholly inside X in both, and in the second series it would carry the run into j+2
     * (its last edge window is X, so head(j+2) does not lead). */
    const uint32_t n_bk = (ch.gc_cols - ch.gc_edge0) / 3;
    for (int which = 0; which < 2; which++) {
        const uint32_t gcol = ch.gc_edge0 + (which ? 2u : (j & 1u)) * n_bk + ch.series_begin / 32 + blk - ch.gc_col0;
        const bool has = r.hb != OG_NO_BUCKET && (which == 0 ? r.head_leader : r.tb != OG_NO_BUCKET);
        const uint32_t b = which == 0 ? r.hb : r.tb;
        const uint32_t hm = __ballot_sync(0xffffffffu, has);
        if (hm == 0) continue;
        const int leader = __ffs(hm) - 1;
        const uint32_t bL = __shfl_sync(0xffffffffu, b, leader);
        const bool unif = __all_sync(0xffffffffu, !has || b == bL) && bL < q.n_buckets;
        if (!unif && has && b >= q.n_buckets) { report_err(ch.err, D_CORRUPT, seg); continue; }
        for (uint32_t c = 0; c < q.n_calls; c++) {
            Part acc = part_empty();
            if (has) acc = edge_stitch(q, ch, r, seg, which, c);
            if (unif) {
                acc = warp_fold(q.calls[c].func, call_ftype(q, c), q.multi != 0, acc, call_has_time(q, c));
                if ((int)lane == leader && acc.ok) store_part(ch.gcells[c], (size_t)bL * ch.gc_cols + gcol, acc);
            } else if (has && acc.ok) store_cell(ch, (int)c, series, b, acc);
        }
    }
}

/* ------------------------------------------------------------------------------------------------------------
 * tagset merge: thread per (group, bucket); series of the group in shard order (CSR), restricted to the chunk
 * ------------------------------------------------------------------------------------------------------------ */
struct GroupP {
    const uint32_t *grp_begin;  /* [n_groups+1] */
    const uint32_t *grp_series; /* series ids sorted by (group, series) */
    uint32_t n_groups;
    Tri dense[OG_MAX_CALLS];    /* [g * n_buckets + b] accumulators (persist across chunks) */
};

__global__ void k_merge_groups(QueryP q, ChunkP ch, GroupP gp) {
    if (ch.flags[0] == 0) return; /* no per-series cell was written */
    size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    size_t total = (size_t)gp.n_groups * q.n_buckets;
    if (idx >= total) return;
    uint32_t g = (uint32_t)(idx / q.n_buckets), b = (uint32_t)(idx % q.n_buckets);
    uint32_t lo = gp.grp_begin[g], hi = gp.grp_begin[g + 1];
    { /* first member >= series_begin */
        uint32_t a = lo, z = hi;
        while (a < z) { uint32_t m = (a + z) >> 1; if (gp.grp_series[m] < ch.series_begin) a = m + 1; else z = m; }
        lo = a;
    }
    if (lo >= hi || gp.grp_series[lo] >= ch.series_end) return;
    { /* one thread per (group, bucket, call): blockIdx.y = call */
        const uint32_t c = blockIdx.y;
        const CallP &cp = q.calls[c];
        Part acc = load_part(gp.dense[c], idx);
        const Tri cells = ch.cells[c];
        /* The fold is strictly sequential in series order (that is the reference's order, reccord_functions.go:730-733),
         * but the loads do not depend on it: fetch a batch of U partials first, so each thread keeps U independent
         * loads in flight.  Threads of a warp own consecutive buckets: every load is a coalesced run of one series row. */
        constexpr int U = 16;
        for (uint32_t i = lo; i < hi; i += U) {
            uint32_t okv[U]; uint64_t vv[U]; int64_t tt[U];
#pragma unroll
            for (int u = 0; u < U; u++) {
                uint32_t ii = i + u;
                uint32_t s = ii < hi ? gp.grp_series[ii] : 0xffffffffu;
                bool in = s < ch.series_end;
                size_t ci = in ? cell_idx(ch, s, b) : 0;
                okv[u] = in ? cells.ok[ci] : 0;
                vv[u] = okv[u] ? cells.val[ci] : 0;
                tt[u] = (okv[u] && cells.tim) ? cells.tim[ci] : 0;
            }
#pragma unroll
            for (int u = 0; u < U; u++) {
                if (!okv[u]) continue;
                Part p; p.ok = 1; p.v = vv[u]; p.t = tt[u];
                group_update(cp.func, cp.out_type == OG_TYPE_INT && cp.func == OG_AGG_COUNT ? OG_TYPE_INT : cp.type, q.multi != 0, acc, p);
            }
        }
        store_part(gp.dense[c], idx, acc);
    }
}

/* OG_GROUP_PER_SERIES: every tagset is one series and the cell matrix already has the dense record's layout, so the merge
 * is elementwise: each cell goes through group_update on an empty accumulator (same value/time rules as the general merge). */
__global__ void k_merge_per_series(QueryP q, ChunkP ch, GroupP gp) {
    const uint32_t c = blockIdx.y;
    const size_t n = (size_t)(ch.series_end - ch.series_begin) * q.n_buckets;
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const CallP &cp = q.calls[c];
    const int ftype = cp.out_type == OG_TYPE_INT && cp.func == OG_AGG_COUNT ? OG_TYPE_INT : cp.type;
    const uint32_t b = (uint32_t)(i % q.n_buckets);
    Part p; p.ok = ch.cells[c].ok[i]; p.v = p.ok ? ch.cells[c].val[i] : 0; p.t = (p.ok && ch.cells[c].tim) ? ch.cells[c].tim[i] : 0;
    Part a; a.v = 0; a.ok = 0; a.t = q.multi ? 0 : q.start + (int64_t)b * q.interval;
    group_update(cp.func, ftype, q.multi != 0, a, p);
    store_part(gp.dense[c], (size_t)ch.series_begin * q.n_buckets + i, a);
}

/* one tagset, order not pinned (no OG_Q_STRICT_ORDER): the per-series cells of a block of OG_MERGE_SB consecutive series are
 * folded in series order by one thread per bucket (coalesced across buckets), and the block partials go to the folded cell
 * matrix (column = block) that k_merge_folded reduces — thousands of threads instead of one per bucket when a shard has many
 * series and few buckets. */
#define OG_MERGE_SB 256u
__global__ void __launch_bounds__(128) k_merge_all_blocks(QueryP q, ChunkP ch, GroupP gp) {
    if (ch.flags[0] == 0) return; /* no per-series cell was written */
    const uint32_t b = blockIdx.x * blockDim.x + threadIdx.x, blk = blockIdx.y, c = blockIdx.z;
    if (b >= q.n_buckets) return;
    const uint32_t nS = ch.series_end - ch.series_begin;
    const uint32_t s0 = blk * OG_MERGE_SB, s1 = min(nS, s0 + OG_MERGE_SB);
    const int func = q.calls[c].func, ftype = call_ftype(q, c);
    const bool multi = q.multi != 0;
    const Tri cells = ch.cells[c];
    Part acc = part_empty();
    constexpr int U = 8;
    for (uint32_t s = s0; s < s1; s += U) {
        uint32_t okv[U]; uint64_t vv[U]; int64_t tt[U];
#pragma unroll
        for (int u = 0; u < U; u++) {
            const bool in = s + u < s1;
            const size_t ci = in ? (size_t)(s + u) * ch.nb + b : 0;
            okv[u] = in ? cells.ok[ci] : 0;
            vv[u] = okv[u] ? cells.val[ci] : 0;
            tt[u] = (okv[u] && cells.tim) ? cells.tim[ci] : 0;
        }
#pragma unroll
        for (int u = 0; u < U; u++) {
            if (!okv[u]) continue;
            Part p; p.ok = 1; p.v = vv[u]; p.t = tt[u];
            group_update(func, ftype, multi, acc, p);
        }
    }
    if (acc.ok) store_part(ch.gcells[c], (size_t)b * ch.gc_cols + blk, acc);
}

/* one tagset: dense[b] (+)= fold over the columns of the folded cell matrix (warp per bucket, grid.y = call; lanes take
 * columns lane, lane+32, ... in order, then a butterfly: a fixed association, so results are reproducible run to run) */
__global__ void k_merge_folded(QueryP q, ChunkP ch, GroupP gp) {
    const uint32_t b = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31, c = blockIdx.y;
    if (b >= q.n_buckets) return;
    const int func = q.calls[c].func, ftype = call_ftype(q, c);
    const bool wt = call_has_time(q, c), multi = q.multi != 0;
    const Tri g = ch.gcells[c];
    Part acc = part_empty();
    const size_t row = (size_t)b * ch.gc_cols;
    for (uint32_t col = lane; col < ch.gc_cols; col += 32) {
        if (!g.ok[row + col]) continue;
        Part p; p.ok = 1; p.v = g.val[row + col]; p.t = wt ? g.tim[row + col] : 0;
        group_update(func, ftype, multi, acc, p);
    }
    acc = warp_fold(func, ftype, multi, acc, wt);
    if (lane == 0 && acc.ok) {
        Part a = load_part(gp.dense[c], b);
        group_update(func, ftype, multi, a, acc);
        store_part(gp.dense[c], b, a);
    }
}

/* dense initialisation: values 0, valid 0, times = window start (single-call selectors) or 0 (RecMeta.Times) */
__global__ void k_init_dense(QueryP q, GroupP gp) {
    size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    size_t total = (size_t)gp.n_groups * q.n_buckets;
    if (idx >= total) return;
    uint32_t b = (uint32_t)(idx % q.n_buckets);
    for (uint32_t c = 0; c < q.n_calls; c++) {
        gp.dense[c].val[idx] = 0; gp.dense[c].ok[idx] = 0;
        if (gp.dense[c].tim) gp.dense[c].tim[idx] = q.multi ? 0 : q.start + (int64_t)b * q.interval;
    }
}

/* merge another shard's dense partial (same geometry) into ours: the cross-shard step for selector aggregates */
__global__ void k_merge_dense(QueryP q, GroupP mine, GroupP other) {
    size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    size_t total = (size_t)mine.n_groups * q.n_buckets;
    if (idx >= total) return;
    for (uint32_t c = 0; c < q.n_calls; c++) {
        const CallP &cp = q.calls[c];
        Part a = load_part(mine.dense[c], idx), p = load_part(other.dense[c], idx);
        group_update(cp.func, cp.func == OG_AGG_COUNT ? OG_TYPE_INT : cp.type, q.multi != 0, a, p);
        store_part(mine.dense[c], idx, a);
    }
}

} // namespace ogpu
