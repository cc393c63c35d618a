/*
 * il_build.cuh — builds the lane-interleaved, length-binned stream copy that k_fused_il reads (once per shard and column).
 *
 *   k_il_scan        per segment: static class (Gorilla stream / packed XOR deltas / not eligible), stream length in words,
 *                    the const-delta time page's (t0, dt), and the sort key (domain, words).  Every eligible page (Gorilla with
 *                    a Full header, or raw) is walked once with ColIter: the OR of the XORs of consecutive values gives the
 *                    delta window lead = clz, trail = ctz, m = 64 - lead - trail (0 when all values are equal).  The packed
 *                    form takes 2 + ceil((rows - 1) * m / 32) words; it is chosen when that is fewer words than the Gorilla
 *                    stream, and always for a raw page.  A page ColIter reports corrupt keeps its stored form, so the query
 *                    reports it exactly as before.  A domain is the set of segments that
 *                    may share a lane group: on regular shards (every series has J segments) segment index j of a block of
 *                    OG_IL_SUPER consecutive series — they cover the same time range, so their windows coincide; otherwise
 *                    the whole shard.  It also checks that every segment index covers one [seg_tmin, seg_tmax] across the
 *                    series of its domain (the folded query path relies on it).
 *   radix sort       (cub::DeviceRadixSort, stable) orders the eligible segments by (domain, words): 32 consecutive entries of
 *                    one domain make a lane group of similar stream lengths.
 *   k_il_assign      sorted position -> (group, lane) slot; writes the per-lane metadata the kernel needs (segment, rows,
 *                    delta window, series, t0, dt) as coalesced arrays.  Packed and Gorilla lanes may share a group.
 *   k_il_group_rows  rows of a group = longest lane + pad, rounded up to the bulk-copy batch.
 *   k_il_repack      word w of lane l -> il[grp_off + w*32 + l], big-endian stream words stored in native order.  A Gorilla
 *                    lane copies its page's stream; a packed lane decodes its page again with ColIter and writes v0 in 64
 *                    bits, then (v_i ^ v_i-1) >> trail in m bits each, MSB first.  Raw pages (float.go:96-99: Gorilla output
 *                    above 90 % of raw) are always packed, with the window of their data (m = 64 at most).
 */
#pragma once
#include "fused_il.cuh"

namespace ogpu {

#define OG_IL_SUPER 4096u      /* series per binning domain (chunks of series are multiples of it when possible) */
#define OG_IL_WORD_BITS 24u    /* sort key = domain << 24 | words */

struct IlScanOut {
    uint32_t *seg_words;    /* [n_segments] stream words incl. pad (0 = not eligible) */
    uint16_t *seg_win;      /* [n_segments] OG_IL_PACKED | lead << 8 | m for SEG_PACKED, else 0 */
    unsigned long long *n_packed; /* [1] SEG_PACKED segments */
    int64_t *seg_t0;        /* [n_segments] */
    uint64_t *seg_dt;
    uint64_t *keys;         /* [n_segments] sort key, ~0 = not eligible */
    uint32_t *vals;         /* [n_segments] = segment id */
    uint32_t *dom_cnt;      /* [n_domains] eligible segments per domain */
    uint32_t *misaligned;   /* [1] set when some segment index covers different time ranges in two series of one domain */
};

/* the window of the XOR deltas of a Full Gorilla or raw page: OR of v_i ^ v_i-1 over the page, walked with ColIter.
 * false: ColIter found the page corrupt, or (m_stop < 64) the window grew to m_stop bits before the last row — the packed form
 * could not be shorter than the page's own stream, so the rest of the walk is skipped */
__device__ inline bool il_delta_window(const uint8_t *page, uint32_t len, uint32_t rows, uint32_t m_stop, uint32_t &lead, uint32_t &m) {
    ColIter it;
    it.init(page, len, OG_TYPE_FLOAT, rows);
    uint64_t prev = 0, acc = 0;
    if (it.err != D_OK || !it.next(prev)) return false;
    for (uint32_t r = 1; r < rows && it.err == D_OK; r++) {
        uint64_t v = 0;
        if (!it.next(v)) return false;
        acc |= v ^ prev; prev = v;
        if ((r & 31) == 0 && m_stop < 64 && acc && 64 - __clzll((long long)acc) - (__ffsll((long long)acc) - 1) >= (int)m_stop) return false;
    }
    if (it.err != D_OK) return false;
    lead = acc ? (uint32_t)__clzll((long long)acc) : 0u;
    m = acc ? 64u - lead - (uint32_t)(__ffsll((long long)acc) - 1) : 0u;
    return true;
}

__global__ void k_il_scan(DirP d, int col, int col_type, uint32_t J, IlScanOut o) {
    uint32_t seg = blockIdx.x * blockDim.x + threadIdx.x;
    if (seg >= d.n_segments) return;
    uint8_t c = SEG_GENERAL; uint32_t nw = 0; int64_t t0 = 0; uint64_t dt = 0; uint16_t win = 0;
    const uint32_t rows = d.seg_rows[seg];
    if (rows >= 2 && rows < (1u << 22) && col_type == OG_TYPE_FLOAT) {
        size_t pi = (size_t)col * d.n_segments + seg, ti = (size_t)d.n_columns * d.n_segments + seg;
        const uint8_t *p = d.data + d.page_off[pi], *t = d.data + d.page_off[ti];
        uint32_t len = d.page_len[pi], tlen = d.page_len[ti];
        /* time page: [32][u32 rows][0x10][t0][uvarint dt][uvarint n-1] */
        TimeDesc td;
        if (len >= 16 && tlen >= 16 && __ldg(p) == 31 && __ldg(t) == 32 && (__ldg(t + 5) >> 4) == 1 && ld_be32(p + 1) == rows &&
            parse_time_page(t, tlen, td) == D_OK && td.kind == 0 && td.delta > 0 && td.delta < (1ull << 40)) {
            const int tag = __ldg(p + 5) >> 4;
            if (tag == 3 && __ldg(p + 6) == 0x10) { /* value page: [31][u32 rows][0x30][0x10][8 B first]... */
                c = SEG_FAST; nw = (len - OG_IL_HDR + 3) / 4 + OG_IL_PAD_WORDS;
            } else if (tag == 0 && len == OG_IL_RAW_HDR + 8 * (size_t)rows) { /* raw page: [31][u32 rows][0x00][rows x 8 B LE] */
                c = SEG_PACKED; nw = 2 * rows + OG_IL_PAD_WORDS; win = OG_IL_PACKED | 64u; /* full 64-bit deltas unless the walk finds a narrower window */
            }
            /* a Gorilla page: the packed form is no shorter from m_stop bits on (2 + ceil((rows-1)*m/32) + pad >= nw) */
            uint32_t m_stop = 64, lead, m;
            if (c == SEG_FAST) {
                const uint32_t T = nw > 2 + OG_IL_PAD_WORDS ? nw - 2 - OG_IL_PAD_WORDS : 0;
                const uint64_t ms = T ? (32ull * (T - 1)) / (rows - 1) + 1 : 0;
                m_stop = ms < 64 ? (uint32_t)ms : 64u;
            }
            if (c != SEG_GENERAL && il_delta_window(p, len, rows, m_stop, lead, m)) {
                const uint32_t pw = 2u + (uint32_t)(((uint64_t)(rows - 1) * m + 31) / 32) + OG_IL_PAD_WORDS;
                if (c == SEG_PACKED || pw < nw) { c = SEG_PACKED; nw = pw; win = (uint16_t)(OG_IL_PACKED | lead << 8 | m); }
            }
            if (nw >= (1u << OG_IL_WORD_BITS)) { c = SEG_GENERAL; nw = 0; win = 0; }
            t0 = td.t0; dt = td.delta;
        }
    }
    o.seg_words[seg] = nw; o.seg_win[seg] = win; o.seg_t0[seg] = t0; o.seg_dt[seg] = dt; o.vals[seg] = seg;
    { /* one atomic per warp */
        const unsigned am = __activemask(), pm = __ballot_sync(am, c == SEG_PACKED);
        if (pm && (threadIdx.x & 31) == (unsigned)(__ffs(am) - 1)) atomicAdd(o.n_packed, (unsigned long long)__popc(pm));
    }
    const uint32_t series = d.seg_series[seg];
    if (J) { /* same time range as segment index j of the domain's first series? */
        const uint32_t ref = d.series_seg_begin[series / OG_IL_SUPER * OG_IL_SUPER] + (seg - d.series_seg_begin[series]);
        if (d.seg_tmin[seg] != d.seg_tmin[ref] || d.seg_tmax[seg] != d.seg_tmax[ref]) *o.misaligned = 1;
    }
    if (c == SEG_GENERAL) { o.keys[seg] = ~0ull; return; }
    const uint32_t dom = J ? (series / OG_IL_SUPER) * J + (seg - d.series_seg_begin[series]) : 0u;
    o.keys[seg] = ((uint64_t)dom << OG_IL_WORD_BITS) | nw;
    atomicAdd(&o.dom_cnt[dom], 1u);
}

struct IlAssign {
    const uint64_t *keys; const uint32_t *segs;    /* sorted */
    const uint32_t *elem_first, *grp_first;        /* [n_domains] first sorted position / first group of each domain */
    const uint32_t *seg_words; const int64_t *seg_t0; const uint64_t *seg_dt; const uint16_t *seg_win;
    uint32_t *lane_seg, *lane_rows, *lane_series, *grp_col; uint16_t *lane_win; int64_t *lane_t0; uint64_t *lane_dt;
    uint32_t n_elig, J, cols_per_super;
};
__global__ void k_il_assign(DirP d, IlAssign a) {
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= a.n_elig) return;
    const uint32_t seg = a.segs[i], dom = (uint32_t)(a.keys[i] >> OG_IL_WORD_BITS);
    const uint32_t rank = i - a.elem_first[dom], g = a.grp_first[dom] + rank / 32;
    const size_t slot = (size_t)g * 32 + (rank & 31);
    a.lane_seg[slot] = seg;
    a.lane_rows[slot] = d.seg_rows[seg];
    a.lane_win[slot] = a.seg_win[seg];
    a.lane_series[slot] = d.seg_series[seg];
    a.lane_t0[slot] = a.seg_t0[seg]; a.lane_dt[slot] = a.seg_dt[seg];
    if ((rank & 31) == 0) a.grp_col[g] = (a.J ? dom / a.J : 0u) * a.cols_per_super + rank / 32;
}

/* rows of every lane group = max over its lanes, rounded up to the bulk-copy batch (one warp per group) */
__global__ void k_il_group_rows(uint32_t n_groups, const uint32_t *lane_seg, const uint32_t *seg_words, uint32_t *grp_rows) {
    uint32_t g = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (g >= n_groups) return;
    uint32_t seg = lane_seg[(size_t)g * 32 + lane];
    uint32_t w = seg != OG_IL_NONE ? seg_words[seg] : 0;
#pragma unroll
    for (int o = 16; o; o >>= 1) w = max(w, __shfl_xor_sync(0xffffffffu, w, o));
    if (lane == 0) grp_rows[g] = (w + OG_IL_B - 1) / OG_IL_B * OG_IL_B;
}

/* the repack (one warp per group; every store is one full 128-byte row) */
__global__ void k_il_repack(DirP d, int col, const uint32_t *lane_seg, const uint16_t *lane_win, const uint64_t *grp_off, const uint32_t *grp_rows,
                            uint32_t n_groups, uint32_t *il) {
    uint32_t g = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (g >= n_groups) return;
    const uint32_t nw = grp_rows[g];
    if (nw == 0) return;
    const size_t slot = (size_t)g * 32 + lane;
    const uint32_t seg = lane_seg[slot];
    const bool live = seg != OG_IL_NONE;
    const uint32_t win = live ? lane_win[slot] : 0u;
    const bool packed = (win & OG_IL_PACKED) != 0;
    /* Gorilla lane: the page's stream bytes s[4w..4w+3] big-endian, from aligned words a = base[w], b = base[w+1] */
    const uint32_t *base = nullptr; uint32_t sh = 0, own_words = 0, a = 0, sel = 0;
    /* packed lane: pending field (pend, its low pbits bits) -> output bits (acc, its high nb bits) */
    ColIter it;
    uint64_t prev = 0, pend = 0, acc = 0; uint32_t pbits = 0, nb = 0, left = 0, mw = 0, tr = 0;
    if (live) {
        const size_t pi = (size_t)col * d.n_segments + seg;
        const uint8_t *page = d.data + d.page_off[pi];
        if (packed) {
            it.init(page, d.page_len[pi], OG_TYPE_FLOAT, d.seg_rows[seg]);
            it.next(prev);
            pend = prev; pbits = 64;
            mw = win & 127u;
            tr = mw ? 64u - ((win >> 8) & 63u) - mw : 0u;
            left = mw ? d.seg_rows[seg] - 1 : 0u; /* m = 0: every delta is empty */
        } else {
            const uint8_t *s = page + OG_IL_HDR;
            base = (const uint32_t *)((uintptr_t)s & ~(uintptr_t)3);
            sh = (uint32_t)((uintptr_t)s & 3);
            own_words = (d.page_len[pi] - OG_IL_HDR + 3) / 4 + OG_IL_PAD_WORDS; /* bytes past the page are the next page or the shard's tail padding */
            a = __ldg(base);
            sel = sh == 0 ? 0x0123u : sh == 1 ? 0x1234u : sh == 2 ? 0x2345u : 0x3456u;
        }
    }
    uint32_t *out = il + grp_off[g] + lane;
    for (uint32_t w = 0; w < nw; w++) {
        uint32_t v = 0;
        if (packed) {
            while (nb < 32) {
                if (pbits == 0) {
                    if (left == 0) break;
                    uint64_t x = 0;
                    it.next(x);
                    pend = (x ^ prev) >> tr; prev = x; pbits = mw; left--;
                }
                const uint32_t k = pbits < 32 ? pbits : 32;
                acc |= ((pend >> (pbits - k)) & (~0ull >> (64 - k))) << (64 - nb - k);
                nb += k; pbits -= k;
            }
            v = (uint32_t)(acc >> 32);
            acc <<= 32; nb = nb > 32 ? nb - 32 : 0;
        } else if (w < own_words) {
            const uint32_t b = __ldg(base + w + 1);
            v = __byte_perm(a, b, sel);
            a = b;
        }
        out[(size_t)w * 32] = v;
    }
}

} // namespace ogpu
