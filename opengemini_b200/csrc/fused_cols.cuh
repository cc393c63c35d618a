/*
 * fused_cols.cuh — K5 for queries over several field columns and/or one WHERE term (configs[2]), column at a time.
 *
 * k_fused_multi walks the rows of a segment once and pulls every column through a generic iterator: a codec switch, a validity
 * test, the call table and the filter are interpreted per row and per column (~540 issue slots per row at configs[2]), and every
 * value costs several unaligned 8-byte loads that touch 32 different sectors per warp instruction.  Here the loops are swapped:
 * one thread still owns one segment, but it walks ONE column at a time in a loop specialised for that page's codec, and columns
 * meet through a per-thread row mask instead of through registers:
 *
 *   pass 0 (only with a WHERE term): the filter's column -> keep bit per row (1024-bit mask in local memory); calls on that
 *          column are accumulated in the same pass;
 *   pass k: every other column of the query: decode, test the row's keep bit, accumulate that column's calls.
 *
 * Every pass walks the same windows (they depend on the time page alone — const-delta here, so row ranges and window boundaries
 * are closed forms / a Bresenham step, not per-row compares) and writes only its own calls' partials: edges for the first and
 * last window of the segment, per-series cells in between — the same outputs k_fused_multi writes, so k_fix_edges and the merges
 * are shared.  Bit streams (Gorilla) are read through a three-word register window refilled with aligned 4-byte loads (one load
 * per 32 bits consumed); Simple8b consumes its word by shifting; bool pages and null bitmaps are read a byte per 8 rows.
 *
 * Eligibility (plan time): every time page of the shard is const-delta or one-row, segments hold <= OG_COLS_MAXROWS rows, the
 * WHERE is at most one compare term, and no column carries more than OG_COLS_MAXMINE calls.  Anything else runs k_fused_multi.
 *
 * Replaces the same reference code as k_fused_multi: readSegmentRecord (tssp_file.go:369) + decodeColumnData (reader.go:674) +
 * FilterByTime (reader.go:754) + FilterByField (reader.go:895-974, functions.go:632: NULL never matches) + aggregateCursor
 * (aggregate_cursor.go:306-356) + the per-window reducers (series_agg_func.gen.go:24-274).
 */
#pragma once
#include "fused_multi.cuh"
#include "fused_il.cuh"
#include <type_traits>

namespace ogpu {

#define OG_COLS_MAXROWS 1024u
#define OG_COLS_MAXMINE 4

/* 64 bits of a big-endian bit stream at any bit position, from cached 32-bit words: wa, wb, wc hold words wi, wi+1, wi+2 (what a
 * 64-bit read at a bit offset inside word wi needs), wd holds word wi+3 — loaded one refill before it is first used, so the load
 * latency overlaps a few records of decoding instead of stalling the read that follows */
struct BitWin {
    const uint32_t *base; uint32_t wa, wb, wc, wd, wi;
    __device__ __forceinline__ uint32_t ldw(uint32_t i) const { return __byte_perm(__ldg(base + i), 0, 0x0123); }
    /* returns the bit offset of `p` inside the aligned word stream */
    __device__ __forceinline__ uint32_t init(const uint8_t *p) {
        const uintptr_t a = (uintptr_t)p;
        base = (const uint32_t *)(a & ~(uintptr_t)3);
        wi = 0; wa = ldw(0); wb = ldw(1); wc = ldw(2); wd = ldw(3);
        return (uint32_t)(a & 3) * 8;
    }
    __device__ __forceinline__ uint64_t peek(uint32_t P) {
        const uint32_t word = P >> 5;
        while (wi != word) { wa = wb; wb = wc; wc = wd; wi++; wd = ldw(wi + 3); } /* a record moves the position by <= 77 bits: <= 3 steps */
        const uint32_t sh = P & 31;
        return ((uint64_t)__funnelshift_l(wb, wa, sh) << 32) | __funnelshift_l(wc, wb, sh);
    }
};

/* simple8b selector -> (values in the word, bits per value) without a table in local memory (simple8b/encoding.go:193-210) */
__device__ __forceinline__ void s8b_sel_packed(unsigned sel, unsigned &n, unsigned &bits) {
    const uint64_t NLO = 0x0a0c0f141e3c78f0ull, NHI = 0x0102030405060708ull; /* 240,120,60,30,20,15,12,10 | 8,7,6,5,4,3,2,1 */
    const uint64_t BLO = 0x0605040302010000ull, BHI = 0x3c1e140f0c0a0807ull; /* 0,0,1,2,3,4,5,6 | 7,8,10,12,15,20,30,60 */
    const unsigned sh = (sel & 7) * 8;
    n = (unsigned)(((sel & 8) ? NHI : NLO) >> sh) & 0xff;
    bits = (unsigned)(((sel & 8) ? BHI : BLO) >> sh) & 0xff;
}

enum { CK_GENERIC = 0, CK_GORILLA = 1, CK_S8B = 2, CK_BITS = 3 };

/* per-thread state of one segment that every column pass shares */
struct ColsSeg {
    uint32_t seg, series, rows, r_lo, r_hi; size_t e;
    int64_t t0, dt; uint64_t dtu;
    uint32_t b_first, rb_first, step_q; uint64_t rem_first, step_r;
};

/* one column of one segment: MODE 0 no WHERE, 1 this is the WHERE column (writes the keep mask), 2 another column (reads it) */
template <int KIND, int MODE, bool SIMPLE>
__device__ __forceinline__ void cols_pass(const QueryP &q, const ChunkP &ch, const ColsSeg &sg, ColIter &it, uint32_t *keep,
                                          int nm, const int (&mc)[OG_COLS_MAXMINE]) {
    /* ---- decoder state in registers ---- */
    BitWin bw; uint32_t P = 0, gend = 0, tr = 0, mb = 64; uint64_t cur = it.cur;       /* Gorilla */
    uint64_t sw = 0, smask = 0, snext = 0; uint32_t sbits = 0, sleft = 0, swords = it.words_left;  /* Simple8b */
    const uint8_t *sp = it.p;
    if (KIND == CK_S8B && swords) snext = ld_be64(sp); /* the next word is always loaded one refill ahead of its use */
    uint32_t bbyte = 0;                                                                  /* bool */
    uint32_t idx = 0;                                                                    /* values consumed */
    if (KIND == CK_GORILLA) { const uint32_t b0 = bw.init(it.p); P = b0; gend = b0 + it.c; }
    auto next_value = [&]() -> uint64_t {
        const uint32_t i = idx++;
        if (KIND == CK_GORILLA) { /* one record of tsm1.FloatArrayDecodeAll (batch_float.go:352-508) */
            if (i == 0) return cur;
            const uint64_t x = bw.peek(P);
            uint32_t used, m;
            if ((x >> 62) == 3) {
                const uint32_t lm = (uint32_t)(x >> 51) & 0x7ff, lead = (lm >> 6) & 0x1f;
                mb = lm & 0x3f;
                if (mb > 0) { if (lead + mb > 64) { it.err = D_CORRUPT; mb = 64; tr = 0; } else tr = 64 - lead - mb; }
                else { tr = 0; mb = 64; }
                used = 13; m = mb;
            } else { used = (x >> 63) ? 2u : 1u; m = (x >> 63) ? mb : 0u; }
            P += used;
            uint64_t y = x << used;
            if (used + m > 64) y = bw.peek(P);
            const uint64_t v = m == 0 ? 0ull : (y >> (64 - m));
            P += m;
            if (P > gend) { it.err = D_CORRUPT; return cur; }
            cur ^= v << tr;
            if (m && cur == OG_UVNAN) it.err = D_CORRUPT; /* the sentinel before the block's value count */
            return cur;
        } else if (KIND == CK_S8B) { /* simple8b words of zig-zag deltas (lib/encoding/int.go:214-265) */
            if (i == 0) return cur;
            while (sleft == 0) {
                if (swords == 0) { it.err = D_CORRUPT; return cur; }
                sw = snext; sp += 8; swords--;
                if (swords) snext = ld_be64(sp);
                unsigned nn; s8b_sel_packed((unsigned)(sw >> 60), nn, sbits);
                sleft = nn;
                if (sbits == 0) { sw = ~0ull; smask = 1; } /* selectors 0/1: runs of the value 1 */
                else smask = (1ull << sbits) - 1;
            }
            const uint64_t z = sw & smask;
            sw >>= sbits; sleft--;
            cur += (uint64_t)zigzag_dec(z);
            return cur;
        } else if (KIND == CK_BITS) { /* MSB-first bit pack (lib/encoding/bool.go:40-61) */
            if ((i & 7) == 0) bbyte = __ldg(it.p + (i >> 3));
            return (uint64_t)((bbyte >> (7 - (i & 7))) & 1);
        } else return it.value();
    };
    /* ---- validity: Full / Empty pages have no bitmap ---- */
    const bool absent = it.kind == ColIter::K_ABSENT;
    const uint8_t *bm = absent ? nullptr : it.h.bitmap;
    const bool all_ok = !absent && !bm && it.h.nil_count == 0;
    const uint32_t bm_off = absent ? 0 : it.h.bm_off;
    uint32_t vb = 0, vb_i = 0xffffffffu;
    auto valid = [&](uint32_t r) -> bool {
        if (!bm) return all_ok;
        const uint32_t b = bm_off + r;
        if ((b >> 3) != vb_i) { vb_i = b >> 3; vb = __ldg(bm + vb_i); }
        return (vb >> (b & 7)) & 1;
    };
    /* the WHERE term (functions.go:632 semantics as term_pass states them: ordered tests pass NaN, = fails it) as an outcome
     * table indexed by (v < c) + 2 (v > c) + 4 (v == c); index 0 = unordered */
    const FilterP &f = q.filter[0];
    const int f_mode = f.type == OG_TYPE_FLOAT ? 0 : (f.type == OG_TYPE_INT && f.const_is_float) ? 1 : f.type == OG_TYPE_BOOL ? 3 : 2;
    const double f_cd = f.const_is_float ? f.fval : (double)f.ival;
    const int64_t f_ci = f.ival;
    const uint32_t f_lt = f.op == OG_OP_LT || f.op == OG_OP_LTE || f.op == OG_OP_NEQ, f_gt = f.op == OG_OP_GT || f.op == OG_OP_GTE || f.op == OG_OP_NEQ;
    const uint32_t f_eq = f.op == OG_OP_LTE || f.op == OG_OP_GTE || f.op == OG_OP_EQ, f_un = f.op != OG_OP_EQ;
    const uint32_t f_tab = f_un | (f_lt << 1) | (f_gt << 2) | (f_eq << 4);
    auto term = [&](uint64_t raw) -> bool {
        uint32_t idx;
        if (f_mode <= 1) {
            double v;
            if (f_mode == 0) v = u2d(raw); else v = (double)(int64_t)raw;
            idx = (uint32_t)(v < f_cd) + 2u * (uint32_t)(v > f_cd) + 4u * (uint32_t)(v == f_cd);
        } else {
            const int64_t v = f_mode == 3 ? (int64_t)(raw != 0) : (int64_t)raw;
            idx = (uint32_t)(v < f_ci) + 2u * (uint32_t)(v > f_ci) + 4u * (uint32_t)(v == f_ci);
        }
        return (f_tab >> idx) & 1;
    };
    int op[OG_COLS_MAXMINE]; /* SIMPLE: 0 count, 1 float sum, 2 integer sum */
#pragma unroll
    for (int j = 0; j < OG_COLS_MAXMINE; j++) {
        const CallP &cp = q.calls[mc[j]];
        op[j] = cp.func == OG_AGG_COUNT ? 0 : cp.type == OG_TYPE_FLOAT ? 1 : 2;
    }

    /* the row loops exist twice: NOBM = Full page (every row valid: no validity test per row), else bitmap / all-null */
    auto run = [&](auto nobm_tag) {
    constexpr bool NOBM = decltype(nobm_tag)::value;
    /* ---- rows before the query range only advance the decoder ---- */
    uint32_t r = 0;
    for (; r < sg.r_lo; r++) if (NOBM || valid(r)) (void)next_value();

    /* ---- windows ---- */
    Part parts[OG_COLS_MAXMINE];
    uint32_t cur_b = sg.b_first, rb = sg.rb_first, w = 0; uint64_t rem = sg.rem_first;
    uint32_t kw = (MODE == 2) ? keep[r >> 5] >> (r & 31) : 0u; /* MODE 2: bit 0 = the keep bit of row r */
    /* SIMPLE (count / sum only): whatever the calls on this column are, they are functions of the count of taken rows and of one
     * running sum — two accumulators per pass instead of one per call */
    const bool fcol = it.type == OG_TYPE_FLOAT;
    uint64_t cnt = 0, isum = 0; double fsum = 0.0;
    while (r <= sg.r_hi) {
        const uint32_t stop = rb < sg.r_hi + 1 ? rb : sg.r_hi + 1;
        if (SIMPLE) { cnt = 0; isum = 0; fsum = 0.0; }
        else {
#pragma unroll
            for (int j = 0; j < OG_COLS_MAXMINE; j++) parts[j] = part_empty();
        }
        for (; r < stop; r++) {
            const bool ok = NOBM || valid(r);
            uint64_t v = 0;
            if (ok) v = next_value();
            bool kp = true;
            if (MODE == 1) {
                kp = ok && term(v);
                kw |= (uint32_t)kp << (r & 31);
                if ((r & 31) == 31) { keep[r >> 5] = kw; kw = 0; }
            } else if (MODE == 2) {
                if ((r & 31) == 0) kw = keep[r >> 5];
                kp = kw & 1; kw >>= 1;
            }
            const bool take = kp && ok;
            if (SIMPLE) { /* count: += 1; sum: sequential add in row order (integerSumReduce / floatSumReduce).  No branch on `take`:
                           * lanes disagree on it row by row.  Adding +0.0 leaves a float sum unchanged bit for bit (a sum that
                           * starts at +0.0 is never -0.0) */
                cnt += (uint64_t)take;
                if (fcol) fsum += take ? u2d(v) : 0.0;
                else isum += take ? v : 0ull;
            } else if (take) {
#pragma unroll
                for (int j = 0; j < OG_COLS_MAXMINE; j++) {
                    if (j >= nm) break;
                    const CallP &cp = q.calls[mc[j]];
                    acc_row(cp.func, cp.type, parts[j], v, sg.t0 + (int64_t)r * sg.dt);
                }
            }
        }
        const bool final = r > sg.r_hi;
#pragma unroll
        for (int j = 0; j < OG_COLS_MAXMINE; j++) {
            if (j >= nm) break;
            if (SIMPLE) { parts[j].t = 0; parts[j].ok = cnt != 0; parts[j].v = op[j] == 0 ? cnt : op[j] == 1 ? d2u(fsum) : isum; }
            if (w == 0) store_part(ch.edges[mc[j]], sg.e, parts[j]);
            else if (final) store_part(ch.edges[mc[j]], sg.e + 1, parts[j]);
            else if (parts[j].ok) store_cell(ch, mc[j], sg.series, cur_b, parts[j]);
        }
        w++;
        if (!final) while (r >= rb) { /* the window that holds row r (a loop: dt may exceed the interval) */
            cur_b++;
            rem += sg.step_r; uint32_t adv = sg.step_q;
            if (rem >= sg.dtu) { rem -= sg.dtu; adv++; }
            rb = (rb > 0xffffffffu - adv) ? 0xffffffffu : rb + adv;
        }
    }
    if (MODE == 1 && (sg.r_hi & 31) != 31) keep[sg.r_hi >> 5] = kw;
    };
    if (!bm && all_ok) run(std::true_type{}); else run(std::false_type{});
    /* a pass that walked to the segment's last row has taken every value of the block: the end-of-page checks of
     * ColIter::finish (every Simple8b slot of every word taken, no word left, exactly n values; RLE runs add up to n) */
    if (sg.r_hi + 1 == sg.rows) {
        if (KIND == CK_GENERIC) it.finish();
        else if (KIND == CK_S8B && (idx != it.h.rows - it.h.nil_count || sleft != 0 || swords != 0)) it.err = D_CORRUPT;
    }
}

template <int MODE, bool SIMPLE>
__device__ __forceinline__ void cols_column(const DirP &d, const QueryP &q, const ChunkP &ch, const ColsSeg &sg, int slot, uint32_t *keep) {
    int mc[OG_COLS_MAXMINE]; int nm = 0;
#pragma unroll
    for (int j = 0; j < OG_COLS_MAXMINE; j++) mc[j] = 0;
    for (uint32_t c = 0; c < q.n_calls; c++) if (q.calls[c].col_slot == slot) {
#pragma unroll
        for (int j = 0; j < OG_COLS_MAXMINE; j++) if (j == nm) mc[j] = (int)c;
        nm++;
    }
    if (MODE != 1 && nm == 0) return; /* a column that only the (absent) filter names */
    const size_t pi = (size_t)q.col_index[slot] * d.n_segments + sg.seg;
    ColIter it;
    it.init(d.data + d.page_off[pi], d.page_len[pi], q.col_type[slot], sg.rows);
    if (it.err != D_OK) { report_err(ch.err, it.err, sg.seg); it.kind = ColIter::K_ABSENT; }
    switch (it.kind) {
    case ColIter::K_F_GORILLA: cols_pass<CK_GORILLA, MODE, SIMPLE>(q, ch, sg, it, keep, nm, mc); break;
    case ColIter::K_I_S8B: cols_pass<CK_S8B, MODE, SIMPLE>(q, ch, sg, it, keep, nm, mc); break;
    case ColIter::K_B_BITS: cols_pass<CK_BITS, MODE, SIMPLE>(q, ch, sg, it, keep, nm, mc); break;
    default: cols_pass<CK_GENERIC, MODE, SIMPLE>(q, ch, sg, it, keep, nm, mc); break;
    }
    if (it.err != D_OK) report_err(ch.err, it.err, sg.seg);
}

#ifndef OG_COLS_MINB
#define OG_COLS_MINB 8 /* blocks/SM the register cap allows; k_fused_cols at configs[2] on an H100 (400 W), ms per 10^9 rows: 8 -> 12.28, 10 -> 12.35-12.54, 12 -> 14.5 */
#endif
template <bool SIMPLE>
__global__ void __launch_bounds__(128, SIMPLE ? OG_COLS_MINB : 4) k_fused_cols(DirP d, QueryP q, ChunkP ch) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    ColsSeg sg;
    sg.seg = ch.seg_begin + i;
    if (sg.seg >= ch.seg_end) return;
    sg.e = 2 * (size_t)(sg.seg - ch.seg_begin);
    sg.rows = d.seg_rows[sg.seg]; sg.series = d.seg_series[sg.seg];
    auto no_rows = [&]() { ch.edge_bucket[sg.e] = OG_NO_BUCKET; ch.edge_bucket[sg.e + 1] = OG_NO_BUCKET; };
    if (d.seg_tmax[sg.seg] < q.tmin || d.seg_tmin[sg.seg] > q.tmax || sg.rows == 0) { no_rows(); return; } /* segment pruning (location.go:276-280) */
    const size_t ti_idx = (size_t)d.n_columns * d.n_segments + sg.seg;
    TimeDesc td;
    const int rc = parse_time_page(d.data + d.page_off[ti_idx], d.page_len[ti_idx], td);
    if (rc != D_OK || (td.kind != 0 && td.kind != 3) || sg.rows > OG_COLS_MAXROWS) { /* the plan promised const-delta pages of <= MAXROWS rows */
        report_err(ch.err, rc != D_OK ? rc : D_CORRUPT, sg.seg); no_rows(); return;
    }
    sg.t0 = td.t0; sg.dtu = td.delta; sg.dt = (int64_t)td.delta;
    /* ---- rows inside [tmin, tmax] (FilterByTime), first window, Bresenham step of the window boundary ---- */
    sg.r_lo = 0; sg.r_hi = sg.rows - 1;
    sg.step_q = 0; sg.step_r = 0; sg.rem_first = 0; sg.rb_first = 0xffffffffu;
    if (sg.dtu == 0) { if (sg.t0 < q.tmin || sg.t0 > q.tmax) { no_rows(); return; } }
    else {
        const double inv_dt = 1.0 / __ull2double_rn(sg.dtu);
        if (sg.t0 < q.tmin) { const uint64_t k = udiv_est((uint64_t)(q.tmin - sg.t0) + sg.dtu - 1, sg.dtu, inv_dt); sg.r_lo = k > sg.rows ? sg.rows : (uint32_t)k; }
        const int64_t t_last = sg.t0 + (int64_t)(sg.rows - 1) * sg.dt;
        if (t_last > q.tmax) { if (q.tmax < sg.t0) sg.r_lo = sg.rows; else sg.r_hi = (uint32_t)udiv_est((uint64_t)(q.tmax - sg.t0), sg.dtu, inv_dt); }
        if (sg.r_lo > sg.r_hi || sg.r_lo >= sg.rows) { no_rows(); return; }
    }
    const int64_t t_lo = sg.t0 + (int64_t)sg.r_lo * sg.dt;
    sg.b_first = bucket_of(t_lo, q.start, q.interval);
    if (sg.dtu != 0) {
        const double inv_dt = 1.0 / __ull2double_rn(sg.dtu);
        const uint64_t ivl = (uint64_t)q.interval;
        const uint64_t sq64 = udiv_est(ivl, sg.dtu, inv_dt);
        sg.step_q = sq64 > 0xffffffffull ? 0xffffffffu : (uint32_t)sq64;
        sg.step_r = ivl - sq64 * sg.dtu;
        /* first row of the next window: ceil((W - t0) / dt), W = start + (b_first + 1) * interval > t_lo >= t0 */
        const uint64_t D = (uint64_t)(q.start + (int64_t)(sg.b_first + 1) * q.interval - sg.t0) + sg.dtu - 1;
        const uint64_t qq = udiv_est(D, sg.dtu, inv_dt);
        sg.rem_first = D - qq * sg.dtu; sg.rb_first = qq > 0xffffffffull ? 0xffffffffu : (uint32_t)qq;
    }
    const uint32_t b_last = bucket_of(sg.t0 + (int64_t)sg.r_hi * sg.dt, q.start, q.interval);
    if (b_last >= q.n_buckets) { report_err(ch.err, D_CORRUPT, sg.seg); no_rows(); return; } /* cannot happen on a validated shard */

    uint32_t keep[OG_COLS_MAXROWS / 32];
    if (q.n_filter) {
        const int fs = q.filter[0].col_slot;
        cols_column<1, SIMPLE>(d, q, ch, sg, fs, keep);
        for (int k = 0; k < (int)q.n_cols; k++) if (k != fs) cols_column<2, SIMPLE>(d, q, ch, sg, k, keep);
    } else {
        for (int k = 0; k < (int)q.n_cols; k++) cols_column<0, SIMPLE>(d, q, ch, sg, k, keep);
    }
    ch.edge_bucket[sg.e] = sg.b_first;
    ch.edge_bucket[sg.e + 1] = b_last == sg.b_first ? OG_NO_BUCKET : b_last;
}

} // namespace ogpu
