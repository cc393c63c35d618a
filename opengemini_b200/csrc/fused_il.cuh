/*
 * fused_il.cuh — K5 for the headline shape: float64 Gorilla pages (tag 3, Full header) and raw float pages (tag 0) with
 * const-delta time pages.  One thread per segment; a warp = one LANE GROUP of 32 segments.
 *
 *   layout    Gorilla decode is serial per stream, so a warp reads 32 different pages.  The shard keeps, next to the pages, a
 *             LANE-INTERLEAVED copy of every eligible stream (built once per shard and column, api.cu ensure_il): the
 *             streams of a group are cut into 32-bit big-endian words and word w of lane l is stored at
 *             il[grp_off + w*32 + l] — one 128-byte row holds word w of all 32 lanes.
 *   binning   groups are formed from segments of the SAME segment index (regular shards: the lanes share one time grid, so
 *             window boundaries coincide) and of SIMILAR STREAM LENGTH (sorted by word count): lanes then advance through
 *             their streams at nearly the same rate, which (a) bounds the padding to the group maximum at ~1 % instead of
 *             ~10 % and (b) lets the whole warp share one window of rows.
 *   staging   rows [f, f+NW) of the group live in a shared-memory ring; ONE lane refills it with cp.async.bulk (TMA, UBLKCP)
 *             in batches of OG_IL_B rows (2 KB contiguous in HBM and in shared memory) that complete on an mbarrier per
 *             batch slot.  No per-lane copies, no per-lane address arithmetic.  Every line of the interleaved copy is read
 *             exactly once, so the copies carry an L2::evict_first policy: they leave L2 first instead of ageing out with
 *             normal priority (DESIGN.md "Staging" has the H100 numbers; an L2 prefetch of later batches ahead of the ring,
 *             cp.async.bulk.prefetch.L2, measured slower than the hint alone at every depth tried).  A lane whose next
 *             OG_IL_K records could touch rows that are not resident yet sits the round out (it only happens when lanes drift apart by more
 *             than ~30 rows, i.e. when binning could not match them).
 *   decode    stateless bit addressing: three LDS.32 at immediate row offsets + two funnel shifts give the 64 stream bits
 *             at bit position q.  q is kept so that the '10' (window reuse) record's payload lands in place:
 *             q = p + 2 - leading  =>  val ^= x & MASK, and the two control bits are tested inside x with one LOP3.
 *   packed    a lane may instead hold its segment as fixed-width XOR deltas (il_build.cuh): the first value in 64 bits, then
 *             (v_i ^ v_i-1) >> trail in m bits each, where [lead, lead + m) is the OR of all the segment's deltas.  The same
 *             path decodes it with q = p - lead, MASK = the window, kfast = m and no control bits (CM = CE = 0): every
 *             record lands in place and the lane never takes slow_record.  Raw pages are always stored so (there is no
 *             separate raw-page kernel), and Gorilla pages whenever that is fewer words — high-entropy data such as G-hi,
 *             whose deltas all sit in one 46-bit window, costs 46 bits a row instead of Gorilla's ~48.6.
 *   reduce    window boundaries are row countdowns derived from the const-delta time page; rounds in which no lane reaches
 *             a boundary run without the per-record test.  Partials stay in registers.  When the query has one tagset and
 *             the lanes share a time grid, the 32 partials of a bucket are folded with warp shuffles and ONE cell per
 *             (bucket, group) is written (gcells; 32x fewer cells, no per-series cell traffic) — interior windows and, when
 *             the group spans more than one bucket, the first/last window of its segments too (tail windows in a column of
 *             their own).  Otherwise the first/last window of a segment goes to the edge arrays (k_fix_edges stitches them
 *             across segments) and each lane writes its own interior cells (cells[series][bucket]), folded in k_merge_* in
 *             strict series order.
 *
 * Replaces for eligible segments: tsm1.FloatArrayDecodeAll (batch_float.go:278-514) + Time.constDeltaDecoding
 * (timestamp.go:190) + FilterByTime (reader.go:754) + getIntervalIndex/reduce (aggregate_cursor.go:306-356) +
 * float{Sum,Min,Max,First,Last}Reduce / *CountReduce (series_agg_func.gen.go:24-274) + the interval-record update of
 * AggTagSetCursor (reccord_functions.go:47-786) for the folded cells.
 */
#pragma once
#include "agg_kernels.cuh"

namespace ogpu {

/* ---- PTX wrappers ---- */
__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ uint32_t opaque(uint32_t x) { asm volatile("mov.u32 %0, %0;" : "+r"(x)); return x; }
template <int OFF> __device__ __forceinline__ uint32_t lds32o(uint32_t a) { uint32_t v; asm volatile("ld.shared.u32 %0, [%1+%2];" : "=r"(v) : "r"(a), "n"(OFF)); return v; }
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) { asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory"); }
/* make the freshly initialised barriers visible to the async proxy (TMA complete_tx) before the first bulk copy is issued */
__device__ __forceinline__ void mbar_init_fence() { asm volatile("fence.mbarrier_init.release.cluster;\nfence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) { asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory"); }
/* TMA bulk copy global -> shared (UBLKCP.S.G); 16-byte aligned addresses, size a multiple of 16; completes on the mbarrier */
__device__ __forceinline__ void bulk_g2s(uint32_t dst, const void *src, uint32_t bytes, uint32_t bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst), "l"(src), "r"(bytes), "r"(bar) : "memory");
}
/* bounded wait (each try_wait suspends up to the hardware time limit): false = the phase never completed.  A bulk copy that
 * cannot complete is a bug or a corrupted directory, never a reason to hang the GPU — callers report D_WATCHDOG and leave. */
__device__ __forceinline__ bool mbar_wait(uint32_t bar, uint32_t parity) {
#pragma unroll 1
    for (uint32_t i = 0; i < (1u << 16); i++) {
        uint32_t ok;
        asm volatile("{\n.reg .pred p;\nmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\nselp.u32 %0, 1, 0, p;\n}" : "=r"(ok) : "r"(bar), "r"(parity) : "memory");
        if (ok) return true;
    }
    return false;
}

enum { FM_COUNT = 1, FM_SUM = 2, FM_MIN = 4, FM_MAX = 8, FM_FIRST = 16, FM_LAST = 32 };
enum { SEG_GENERAL = 0, SEG_FAST = 1, SEG_PACKED = 2 }; /* static per-segment classes (k_il_scan): general kernel / Gorilla stream / fixed-width XOR deltas */

#ifndef OG_FAST_THREADS
#define OG_FAST_THREADS 128
#endif
#ifndef OG_FAST_MAXREG
#define OG_FAST_MAXREG 80 /* registers are granted in steps of 8 per thread: 80 lets six 128-thread blocks share an SM, 88 only five */
#endif
#ifndef OG_IL_NW
#define OG_IL_NW 64u            /* ring rows (words per lane resident) */
#endif
#ifndef OG_IL_B
#define OG_IL_B 16u             /* rows per bulk copy (2 KB) */
#endif
#ifndef OG_IL_K
#define OG_IL_K 10u             /* records per round.  k_fused_il at configs[1] on an H100 (700 W), evict-first ring copies,
                                   ms: 8 -> 11.73, 10 -> 11.74, 12 -> 11.77 (8 and 10 within 0.1 %) */
#endif
#ifndef OG_IL_UNROLL
#define OG_IL_UNROLL 2 /* two pairs per loop trip rather than the fully unrolled round, which is hard on the instruction cache */
#endif
#define OG_IL_NB (OG_IL_NW / OG_IL_B)
#define OG_IL_ROWS (OG_IL_NW + 2u) /* + 2 mirror rows that repeat ring rows 0,1 so that three consecutive rows never wrap */
#define OG_IL_PAD_WORDS 6u      /* words appended to every stream: the decoder may touch 77 + 64 + 32 bits past the last record */
#define OG_IL_HDR 7u            /* page = [31][rows u32][0x30][0x10] | stream: first value 8 B BE, records... */
#define OG_IL_RAW_HDR 6u        /* page = [31][rows u32][0x00] | rows x 8 B LE */
#define OG_IL_NONE 0xffffffffu
/* lane_win of a packed lane: OG_IL_PACKED | lead << 8 | m (lead <= 63, m <= 64); 0 = Gorilla stream */
#define OG_IL_PACKED 0x8000u
/* bits past q that the next K records may touch: K records of <= 77 bits, q = p - sr with sr <= 29, the '11' header (13),
 * one 64-bit fetch and the word rounding of the three-row read.  A packed lane stays inside it for K >= 2: q = p - lead with
 * lead <= 63 and K fields of <= 64 bits, so K*64 + 63 + 64 + 64 bits past q */
#define OG_IL_LOOKBITS (77u * OG_IL_K + 29u + 13u + 64u + 64u)
static_assert(OG_IL_K >= 2, "packed lanes: K*64 + 63 + 128 <= OG_IL_LOOKBITS needs K >= 2");
static_assert(OG_IL_NW % OG_IL_B == 0 && (OG_IL_NW & (OG_IL_NW - 1)) == 0, "ring geometry");
static_assert(OG_IL_NW - OG_IL_B > (OG_IL_LOOKBITS + 31u) / 32u + 2u, "ring too small for the round length: the slowest lane could not proceed");

/* lane-interleaved stream copy of one column (owned by the shard, built lazily by ensure_il) */
struct IlP {
    const uint32_t *words;       /* il[grp_off[g] + row*32 + lane] */
    const uint64_t *grp_off;     /* [n_groups] in words (multiple of 32: rows are 128-byte aligned) */
    const uint32_t *grp_rows;    /* [n_groups] rows of the group (multiple of OG_IL_B), 0 = no lane */
    const uint32_t *grp_col;     /* [n_groups] column of the group in the folded cell matrix (rank inside its segment index) */
    const uint32_t *lane_seg;    /* [n_groups*32] segment of every lane slot, OG_IL_NONE = empty */
    const uint32_t *lane_rows;   /* rows of the segment */
    const uint16_t *lane_win;    /* OG_IL_PACKED | lead << 8 | m for a packed lane, 0 for a Gorilla stream */
    const uint32_t *lane_series; /* series index of the segment */
    const int64_t *lane_t0;      /* const-delta time page: t(r) = t0 + r*dt */
    const uint64_t *lane_dt;
};

/* floor(a / b) for a < 2^63 through a double-precision estimate and an exact 64-bit correction (a handful of instructions
 * instead of the ~150 of the generic 64-bit division; the segment prologue needs six of them).  inv_b = 1.0 / (double)b. */
__device__ __forceinline__ uint64_t udiv_est(uint64_t a, uint64_t b, double inv_b) {
    const double qd = __ull2double_rn(a) * inv_b;
    if ((a >> 63) || !(qd < 1125899906842624.0)) return a / b; /* quotient >= 2^50: the estimate could be off by more than a few units */
    uint64_t q = (uint64_t)qd;
    uint64_t r = a - q * b;
    if ((int64_t)r < 0) { do { q--; r += b; } while ((int64_t)r < 0); }
    else while (r >= b) { q++; r -= b; }
    return q;
}

/* 64 bits of the stream at bit position p: ring rows (p>>5), +1, +2 of the lane's column */
__device__ __forceinline__ uint64_t fetch64(uint32_t col, uint32_t p) {
    uint32_t a = col + ((p << 2) & ((OG_IL_NW - 1) << 7)); /* ((p >> 5) % NW) * 128 */
    uint32_t a0 = lds32o<0>(a), a1 = lds32o<128>(a), a2 = lds32o<256>(a);
    uint32_t hi = __funnelshift_l(a1, a0, p), lo = __funnelshift_l(a2, a1, p); /* shift amount taken mod 32 */
    return ((uint64_t)hi << 32) | lo;
}

/* fold the 32 lanes' partials of one bucket (per-window counts fit 32 bits: one REDUX; float sums: a butterfly of adds, the
 * same association in every lane; float min/max without a carried time: a butterfly of strict compares; selectors that
 * carry a time: warp_fold with the tagset tie-break rules) */
__device__ __forceinline__ Part fold32(int func, int type, bool multi, Part p, bool with_time) {
    constexpr uint32_t FULL = 0xffffffffu;
    if (func == OG_AGG_COUNT) { p.v = __reduce_add_sync(FULL, p.ok ? (uint32_t)p.v : 0u); p.ok = p.v != 0; return p; }
    if (type == OG_TYPE_FLOAT && func == OG_AGG_SUM) {
        double s = p.ok ? u2d(p.v) : 0.0;
#pragma unroll
        for (int o = 16; o; o >>= 1) s += __shfl_xor_sync(FULL, s, o);
        p.ok = __any_sync(FULL, p.ok != 0); p.v = d2u(s); return p;
    }
    if (type == OG_TYPE_FLOAT && !with_time && (func == OG_AGG_MIN || func == OG_AGG_MAX)) { /* update*Column{Min,Max}Impl (reccord_functions.go:586-660) */
        double v = u2d(p.v); uint32_t ok = p.ok;
#pragma unroll
        for (int o = 16; o; o >>= 1) {
            const double ov = __shfl_xor_sync(FULL, v, o); const uint32_t ook = __shfl_xor_sync(FULL, ok, o);
            const bool keep = ok && (func == OG_AGG_MIN ? v <= ov : v >= ov);
            if (ook && !keep) v = ov;
            ok |= ook;
        }
        p.v = d2u(v); p.ok = ok; return p;
    }
    return warp_fold(func, type, multi, p, with_time);
}

#define OG_IL_WCAP 24u /* windows of one segment a folding warp accumulates in shared memory; segments that span more run unfolded */
/* dynamic shared memory per warp for the window accumulators of a folding warp: n_calls x WCAP x {u64 value, i64 time, u8 valid} */
__host__ __device__ inline uint32_t il_acc_bytes(uint32_t n_calls, bool times) { return OG_IL_WCAP * n_calls * (times ? 17u : 9u) + 8u & ~7u; }

template <int FM, bool TIMES, bool FOLD>
__global__ void __maxnreg__(OG_FAST_MAXREG) k_fused_il(QueryP q, ChunkP ch, IlP il, uint32_t grp_begin, uint32_t grp_end) {
    constexpr uint32_t NW = OG_IL_NW, B = OG_IL_B, NB = OG_IL_NB, K = OG_IL_K;
    constexpr uint32_t FULL = 0xffffffffu;
    constexpr uint32_t WPB = OG_FAST_THREADS / 32;
    constexpr int UNR = OG_IL_UNROLL;
    __shared__ __align__(128) uint32_t s_win[WPB * OG_IL_ROWS * 32];
    __shared__ __align__(8) uint64_t s_bar[WPB * NB];
    extern __shared__ __align__(8) uint8_t s_acc[]; /* FOLD: WPB x il_acc_bytes */

#ifdef OG_IL_STATS
    const long long st_clk0 = clock64();
    long long st_wait = 0; /* cycles spent waiting for ring batches to land */
#endif
    const uint32_t lane = threadIdx.x & 31;
    /* warp-uniform values are produced by warp reductions so that the compiler keeps them (and everything derived from them:
     * ring/barrier addresses, batch counters) in uniform registers — the bulk-copy instructions take uniform operands */
    const uint32_t wid = __reduce_max_sync(FULL, threadIdx.x >> 5);
    const uint32_t grp = grp_begin + blockIdx.x * WPB + wid;
    if (grp >= grp_end) return;
    const uint32_t rows_w = __reduce_max_sync(FULL, il.grp_rows[grp]);
    if (rows_w == 0) return;
    const size_t slot = (size_t)grp * 32 + lane;
    const uint32_t seg = il.lane_seg[slot];
    /* a lane group that straddles two chunks runs in both, with complementary lanes */
    bool active = seg != OG_IL_NONE && seg >= ch.seg_begin && seg < ch.seg_end;
    if (!__any_sync(FULL, active)) return;
    const size_t e = 2 * (size_t)(seg - ch.seg_begin);

    uint32_t rows = 0, series = 0, r_lo = 0, r_hi = 0, lwin = 0;
    int64_t t0 = 0, dt = 1; uint64_t dtu = 1; double inv_dt = 1.0;
    const double inv_iv = 1.0 / __ull2double_rn((uint64_t)q.interval);
    if (active) {
        rows = il.lane_rows[slot]; lwin = il.lane_win[slot]; series = il.lane_series[slot];
        t0 = il.lane_t0[slot]; dtu = il.lane_dt[slot]; dt = (int64_t)dtu;
        inv_dt = 1.0 / __ull2double_rn(dtu);
        /* rows inside [tmin, tmax] (FilterByTime) */
        r_lo = 0; r_hi = rows - 1;
        if (t0 < q.tmin) { uint64_t k = udiv_est((uint64_t)(q.tmin - t0) + dtu - 1, dtu, inv_dt); r_lo = k > rows ? rows : (uint32_t)k; }
        { int64_t t_last = t0 + (int64_t)(rows - 1) * dt; if (t_last > q.tmax) { if (q.tmax < t0) r_lo = rows; else r_hi = (uint32_t)udiv_est((uint64_t)(q.tmax - t0), dtu, inv_dt); } }
        /* rows in range outside the buckets [0, n_buckets): cannot happen on a validated shard, and must never become a stray
         * cell store (the lane leaves as if it had no rows) */
        const uint64_t span = (uint64_t)q.n_buckets * (uint64_t)q.interval;
        const bool outside = r_lo <= r_hi && r_lo < rows &&
                             ((uint64_t)(t0 + (int64_t)r_lo * dt - q.start) >= span || (uint64_t)(t0 + (int64_t)r_hi * dt - q.start) >= span);
        if (outside) report_err(ch.err, D_CORRUPT, seg);
        if (r_lo > r_hi || r_lo >= rows || outside) { *(uint2 *)(ch.edge_bucket + e) = make_uint2(OG_NO_BUCKET, OG_NO_BUCKET); active = false; }
    }
    if (!__any_sync(FULL, active)) return;

    /* ---- the warp's ring and its batch barriers ---- */
    const uint32_t win = smem_u32(s_win) + wid * (OG_IL_ROWS * 128);
    const uint32_t col = opaque(win + lane * 4);
    const uint32_t bar0 = smem_u32(s_bar) + wid * (NB * 8);
    if (lane == 0) {
#pragma unroll
        for (uint32_t i = 0; i < NB; i++) mbar_init(bar0 + i * 8, 1);
        mbar_init_fence();
    }
    __syncwarp();
    const uint32_t total_b = rows_w / B;
    uint64_t goff = il.grp_off[grp];
    goff = ((uint64_t)__reduce_max_sync(FULL, (uint32_t)(goff >> 32)) << 32) | __reduce_max_sync(FULL, (uint32_t)goff);
    const uint32_t *gsrc = il.words + goff;
    uint32_t issued_b = 0, ready_b = 0; /* warp-uniform: batches issued / known complete */
    uint32_t hung = 0;                  /* warp-uniform watchdog code: 1 a batch never landed, 2 the round limit was hit */
    /* every lane calls issue(); one elected lane performs it.  The batch index goes through a warp reduction so that slot, ring,
     * barrier and source addresses are uniform-register arithmetic (the bulk copy takes uniform operands; per-thread values would
     * make the compiler wrap it in a broadcast loop).  The copies go to L2 under an evict-first policy ("staging" at the head of
     * this file); its operands are immediates, so the compiler folds the policy into a constant in uniform registers */
    uint64_t pol;
    asm("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(pol));
    auto issue = [&](uint32_t k_any) {
        const uint32_t k = __reduce_max_sync(FULL, k_any);
        const uint32_t s = k % NB, dst = win + s * (B * 128), bar = bar0 + s * 8;
        const uint32_t *src = gsrc + (size_t)k * (B * 32);
        if (s == 0) /* slot 0 also refreshes the two mirror rows behind the ring */
            asm volatile("{\n.reg .pred p;\nelect.sync _|p, 0xffffffff;\n@p mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;\n"
                         "@p cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%2], [%3], %4, [%0], %6;\n"
                         "@p cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%5], [%3], 256, [%0], %6;\n}"
                         ::"r"(bar), "r"(B * 128 + 256u), "r"(dst), "l"(src), "r"(B * 128), "r"(win + NW * 128), "l"(pol) : "memory");
        else
            asm volatile("{\n.reg .pred p;\nelect.sync _|p, 0xffffffff;\n@p mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;\n"
                         "@p cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%2], [%3], %1, [%0], %4;\n}"
                         ::"r"(bar), "r"(B * 128), "r"(dst), "l"(src), "l"(pol) : "memory");
    };
    {
        const uint32_t first = total_b < NB ? total_b : NB;
        for (uint32_t k = 0; k < first; k++) issue(k);
        issued_b = first;
    }

    /* ---- window bookkeeping: bucket of row r_lo, first row of the next bucket (rb), Bresenham advance of rb ---- */
    uint32_t cur_b = 0, rb = 0xffffffffu, step_q = 0; uint64_t rem = 0, step_r = 0;
    if (active) {
        const int64_t t_lo = t0 + (int64_t)r_lo * dt;
        cur_b = (uint32_t)udiv_est((uint64_t)(t_lo - q.start), (uint64_t)q.interval, inv_iv);
        const uint64_t ivl = (uint64_t)q.interval;
        const uint64_t sq64 = udiv_est(ivl, dtu, inv_dt);
        step_q = sq64 > 0xffffffffull ? 0xffffffffu : (uint32_t)sq64;
        step_r = ivl - sq64 * dtu;
        /* rb = ceil((W - t0)/dt), W = start + (cur_b+1)*interval > t_lo >= t0 */
        uint64_t D = (uint64_t)(q.start + (int64_t)(cur_b + 1) * q.interval - t0) + dtu - 1;
        uint64_t qq = udiv_est(D, dtu, inv_dt); rem = D - qq * dtu; rb = qq > 0xffffffffull ? 0xffffffffu : (uint32_t)qq;
    }

    /* ---- folding: the lanes share a time grid (same first row, cadence and row range), so a bucket means the same window to all of
     * them and the segment spans at most WCAP of them.  Lanes may still reach a window at different moments (streams of different
     * entropy drift apart): interior windows are therefore accumulated per bucket in shared memory — whoever closes a window adds
     * its partial, lanes that close the same window in the same step are folded with shuffles first — and written to the folded
     * cell matrix once, when the whole group is done.
     *
     * Edge windows: the first and last window of a segment may continue in the neighbouring segments of its series.  When the
     * group's rows span more than one bucket (b_end > b0), the lanes' head windows all lie in bucket b0 and their tail windows
     * all in b_end, so they are accumulated like interior windows: the head in column gcol (slot 0), the tail in the group's
     * TAIL column gc_tail0 + gcol (slot b_end - b0).  Tails need columns of their own: group (j, r) has its tail in the bucket
     * of the head of group (j+1, r), same column r.  Heads (and tails) of one column never meet in a bucket because segment
     * index j covers one time range in every series of the binning domain (the plan folds only such shards) and those ranges
     * are disjoint and ascending in j: tail(j) <= head(j+1) < tail(j+1).  A group inside one bucket (a window spanning three or
     * more segments) and groups whose lanes disagree (uni false) write their edges to ch.edges for k_fix_edges_fold, and flag
     * it.  Mixing the two is exact: a segment folded here has no edge_bucket entries, which the stitch reads as "no rows in
     * range", so its neighbour leads a run of its own and the two partials of the bucket meet in k_merge_folded through
     * group_update.  Count, sum, min and max are associative there; for selectors that carry a time the part of a series in
     * its tail (earlier times) and the part in the next segment's head (later times) are ordered by time, and group_update
     * picks the earlier time on equal values (first/last: the earlier/later time), exactly what the ordered stitch picks. ---- */
    bool uni = false; uint32_t b0 = 0, b_end = 0;
    uint64_t *acc_v = nullptr; int64_t *acc_t = nullptr; uint8_t *acc_k = nullptr;
    if (FOLD) {
        const int leader = __ffs(__ballot_sync(FULL, active)) - 1;
        /* every lane executes every shuffle (no short-circuit between them) */
        const int64_t t0L = __shfl_sync(FULL, t0, leader); const uint64_t dtL = __shfl_sync(FULL, dtu, leader);
        const uint32_t loL = __shfl_sync(FULL, r_lo, leader), hiL = __shfl_sync(FULL, r_hi, leader);
        b0 = __shfl_sync(FULL, cur_b, leader);
        const bool same = t0 == t0L && dtu == dtL && r_lo == loL && r_hi == hiL;
        const uint32_t b_last = active ? (uint32_t)udiv_est((uint64_t)(t0 + (int64_t)r_hi * dt - q.start), (uint64_t)q.interval, inv_iv) : b0;
        uni = __all_sync(FULL, !active || (same && b_last - b0 < OG_IL_WCAP));
        if (uni) {
            b_end = __reduce_max_sync(FULL, active ? b_last : 0u);
            const uint32_t nacc = OG_IL_WCAP * q.n_calls;
            uint8_t *base = s_acc + (size_t)wid * il_acc_bytes(q.n_calls, TIMES);
            acc_v = (uint64_t *)base; acc_t = (int64_t *)(base + (size_t)nacc * 8); acc_k = base + (size_t)nacc * (TIMES ? 16 : 8);
            for (uint32_t i = lane; i < nacc; i += 32) acc_k[i] = 0;
            __syncwarp();
        }
    }
    const uint32_t gcol = FOLD ? il.grp_col[grp] - ch.gc_col0 : 0;
    /* edge windows folded in the warp as well (head in slot 0, tail in slot b_end - b0; see "edge windows" above) */
    const bool fold_edges = FOLD && uni && b_end > b0;

    /* ---- per-window partials ---- */
    double sum = 0.0, mn = 0.0, mx = 0.0; uint64_t fi = 0, lastv = 0;
    uint32_t n_mn = 0, n_mx = 0;  /* countdown value at the extreme row (row = stop - countdown) */
    uint32_t w_row0 = r_lo;       /* first row of the open window */
    bool head_done = false; uint32_t head_b = OG_NO_BUCKET;
    uint32_t stop = 0, n_ev = 0;
    auto part_of = [&](int func, uint32_t cnt) -> Part {
        Part pp; pp.ok = cnt != 0; pp.v = 0; pp.t = 0;
        switch (func) {
        case OG_AGG_COUNT: pp.v = cnt; break;
        case OG_AGG_SUM: if (FM & FM_SUM) pp.v = d2u(sum); break;
        case OG_AGG_MIN: if (FM & FM_MIN) { pp.v = d2u(mn); if (TIMES) pp.t = t0 + (int64_t)(stop - n_mn) * dt; } break;
        case OG_AGG_MAX: if (FM & FM_MAX) { pp.v = d2u(mx); if (TIMES) pp.t = t0 + (int64_t)(stop - n_mx) * dt; } break;
        case OG_AGG_FIRST: if (FM & FM_FIRST) { pp.v = fi; pp.t = t0 + (int64_t)w_row0 * dt; } break;
        default: if (FM & FM_LAST) { pp.v = lastv; pp.t = t0 + (int64_t)(stop - 1) * dt; } break;
        }
        return pp;
    };
    /* the window [w_row0, stop) of a lane at an event: 0 head edge, 1 tail edge, 2 an interior window */
    auto kind_of = [&]() -> int { return !head_done ? 0 : stop > r_hi ? 1 : 2; };
    auto flush_lane = [&](int kind) { /* this lane alone: edges, or its own cell of the per-series matrix */
        const uint32_t cnt = stop - w_row0;
#pragma unroll 1
        for (uint32_t c = 0; c < q.n_calls; c++) { /* rolled on purpose: this path runs once per window, keep it small */
            const Part pp = part_of(q.calls[c].func, cnt);
            if (kind == 2) { if (pp.ok) store_cell(ch, (int)c, series, cur_b, pp); }
            else store_part(ch.edges[c], e + kind, pp);
        }
        if (kind == 0) { head_done = true; head_b = cur_b; }
    };
    /* folding warp, every lane takes part: `ev` lanes that close an interior window add it to the bucket's accumulator */
    auto flush_fold = [&](bool ev) {
        uint32_t pend = __ballot_sync(FULL, ev);
#pragma unroll 1
        while (pend) { /* one pass per distinct bucket closed in this step (one in lockstep) */
            const int leader = __ffs(pend) - 1;
            const uint32_t bL = __shfl_sync(FULL, cur_b, leader);
            const bool mine = ev && cur_b == bL;
            const uint32_t cnt = mine ? stop - w_row0 : 0;
            const uint32_t w = bL - b0;
#pragma unroll 1
            for (uint32_t c = 0; c < q.n_calls; c++) {
                const int func = q.calls[c].func, ftype = func == OG_AGG_COUNT ? OG_TYPE_INT : q.calls[c].type;
                const bool wt = func >= OG_AGG_MIN && !(q.multi && func <= OG_AGG_MAX);
                Part pp = fold32(func, ftype, q.multi != 0, part_of(func, cnt), wt);
                if ((int)lane == leader && pp.ok) {
                    const uint32_t i = c * OG_IL_WCAP + w;
                    Part a; a.ok = acc_k[i]; a.v = a.ok ? acc_v[i] : 0; a.t = (TIMES && a.ok) ? acc_t[i] : 0;
                    group_update(func, ftype, q.multi != 0, a, pp);
                    acc_v[i] = a.v; acc_k[i] = 1; if (TIMES) acc_t[i] = a.t;
                }
            }
            pend &= ~__ballot_sync(FULL, mine);
        }
        __syncwarp();
    };

    /* ---- decode state ----
     * p = stream bit position of the next record; q = p - sr is what the loop carries, sr = leading - 2 of the open window, so
     * that fetch64(q) holds the '10' payload in place under MASK and the control bits at bits (31-sr, 30-sr) of its high word:
     * '10' <=> ((xhi & CM) ^ CE) == 0 with CM = 3 << k, CE = 2 << k (one LOP3 with a predicate result).  Windows with leading < 2
     * cannot be tested in place (slowwin): CM = 0, CE = 1 never passes, so they, '0' and '11' records take the general path.
     * A finished or empty lane has CM = CE = 0, MASK = 0, kfast = 0: it idles on the fast path. */
    uint32_t qp = 0, sr = 0, kfast = 0, CM = 0, CE = 0, m = 64, tr = 0, bad = 0; uint64_t MASK = 0;
    bool done = !active;
    uint64_t val = 0;

    /* first batch must land before the first value is read */
#ifdef OG_IL_STATS
    long long st_w0 = clock64();
#endif
    if (issued_b && !mbar_wait(bar0, 0)) hung = 1; else ready_b = issued_b ? 1 : 0;
#ifdef OG_IL_STATS
    st_wait += clock64() - st_w0;
#endif
    if (active && !hung) {
        val = fetch64(col, 0); qp = 64; /* first value: 64 raw bits */
        if (lwin & OG_IL_PACKED) { /* m-bit deltas of the window [lead, lead + m): in place at q = p - lead, no control bits */
            const uint32_t lead = (lwin >> 8) & 63u, mw = lwin & 127u;
            qp = 64 - lead; kfast = mw;
            MASK = mw ? (~0ull >> (64 - mw)) << (64 - lead - mw) : 0ull; /* m = 0: a constant segment, the lane never moves */
        } else { CM = 0; CE = 1; } /* Gorilla, no window yet: the first record takes the general path */
    }

    /* ---- row events: skip rows before r_lo, window boundaries, end at r_hi ---- */
    bool skipping = r_lo > 0;
    stop = skipping ? r_lo : (rb < r_hi + 1 ? rb : r_hi + 1); /* row index of the next event */
    n_ev = stop;                                            /* rows until the next event (row 0 is current) */
    if (!skipping) { fi = val; mn = mx = u2d(val); n_mn = n_mx = n_ev; }
    if (done) n_ev = 0xffffffffu;

    auto retire = [&]() { done = true; n_ev = 0xffffffffu; CM = 0; CE = 0; MASK = 0; kfast = 0; };
    auto advance = [&]() { /* bookkeeping of a lane at an event, after its flush */
        bool fin = false;
        if (skipping) { skipping = false; sum = 0.0; }
        else {
            fin = stop > r_hi;
            sum = 0.0;
            if (!fin) while (stop >= rb) { /* advance to the window that contains row `stop` (a loop: dt may exceed the interval) */
                cur_b++;
                rem += step_r; uint32_t adv = step_q;
                if (rem >= dtu) { rem -= dtu; adv++; }
                rb = (rb > 0xffffffffu - adv) ? 0xffffffffu : rb + adv;
            }
        }
        if (fin) retire();
        else {
            w_row0 = stop;
            uint32_t nstop = rb < r_hi + 1 ? rb : r_hi + 1;
            n_ev = nstop - stop; stop = nstop;
            fi = val; mn = mx = u2d(val); n_mn = n_mx = n_ev; /* the first value of a window seeds min/max/first (column_util.go:190-278) */
        }
    };
    auto slow_record = [&]() { /* '0', '11', or '10' on a window that cannot be tested in place (batch_float.go:352-508) */
        uint32_t p = qp + sr;
        const uint64_t x = fetch64(col, p);
        const uint32_t ctrl = (uint32_t)(x >> 62);
        if (ctrl < 2) { qp += 1; return; } /* '0': same value */
        if (ctrl == 3) {                   /* '11': 5 bits leading, 6 bits meaningful */
            const uint32_t lm = (uint32_t)(x >> 51) & 0x7ff;
            uint32_t lead = lm >> 6; m = lm & 0x3f;
            if (m == 0) { m = 64; tr = 0; lead = 0; }
            else { if (lead + m > 64) { if (!done) bad = 1; lead = 0; m = 64; } tr = 64 - lead - m; }
            p += 13;
            const bool slowwin = lead < 2;
            sr = slowwin ? 0 : lead - 2;
            CM = slowwin ? 0u : 3u << (30 - sr); CE = slowwin ? 1u : 2u << (30 - sr);
            kfast = 2 + m;
            MASK = (m == 64 ? ~0ull : ((1ull << m) - 1)) << tr;
        } else p += 2;
        const uint64_t y = fetch64(col, p);
        const uint64_t sig = m == 64 ? y : (y >> (64 - m));
        p += m;
        val ^= sig << tr;
        qp = p - sr;
    };
    auto accumulate = [&](uint32_t k_in_run) { /* the current row; n_ev counts down once per run of records, k_in_run is the offset inside it */
        if (FM & FM_SUM) sum = sum + u2d(val);
        if (FM & FM_MIN) { if (mn > u2d(val)) { mn = u2d(val); if (TIMES) n_mn = n_ev - k_in_run; } }
        if (FM & FM_MAX) { if (mx < u2d(val)) { mx = u2d(val); if (TIMES) n_mx = n_ev - k_in_run; } }
        if (FM & FM_LAST) lastv = val;
    };
    auto record = [&](uint32_t k_in_run) {
        accumulate(k_in_run);
        const uint64_t x = fetch64(col, qp); /* next record */
        const bool slow = (((uint32_t)(x >> 32) & CM) ^ CE) != 0;
        if (slow) slow_record();
        else { val ^= x & MASK; qp += kfast; } /* '10' with the window in place, raw delta, or an idle lane */
    };
    /* two records with both fetches issued up front: record k+1 starts kfast bits after record k when k is an in-place '10'
     * (it nearly always is), so its 64 bits can be loaded before k has been tested — the two shared-memory round trips overlap
     * instead of forming one dependent chain per record.  A wrong guess costs a re-fetch on the general path. */
    auto record2 = [&](uint32_t k_in_run) {
        const uint64_t x0 = fetch64(col, qp), x1 = fetch64(col, qp + kfast);
        accumulate(k_in_run);
#ifdef OG_IL_REC2B
        uint64_t x1b = x1;
        if ((((uint32_t)(x0 >> 32) & CM) ^ CE) != 0) { slow_record(); x1b = fetch64(col, qp); } /* wrong guess: fetch the second record again */
        else { val ^= x0 & MASK; qp += kfast; }
        accumulate(k_in_run + 1);
        if ((((uint32_t)(x1b >> 32) & CM) ^ CE) != 0) slow_record();
        else { val ^= x1b & MASK; qp += kfast; }
#else
        if ((((uint32_t)(x0 >> 32) & CM) ^ CE) != 0) { slow_record(); record(k_in_run + 1); return; }
        val ^= x0 & MASK; qp += kfast;
        accumulate(k_in_run + 1);
        if ((((uint32_t)(x1 >> 32) & CM) ^ CE) != 0) slow_record();
        else { val ^= x1 & MASK; qp += kfast; }
#endif
    };

    /* Rounds.  Every round the slowest live lane decodes K records, so 32 lanes finish within 32 * (rows / K + 1) eventful rounds.
     * The common round — every lane resident, no window boundary within K records — costs two warp reductions and a handful of
     * uniform compares on top of the K records; everything else (events, lanes that drifted ahead of the ring) is the rare path. */
    uint32_t rounds_left = hung ? 0u : 40u * (__reduce_max_sync(FULL, rows) / K + 8u);
#ifdef OG_IL_STATS
    uint32_t st_common = 0, st_rare = 0, st_sit = 0, st_notgo = 0;
    const long long st_pro = clock64() - st_clk0; /* prologue: warp start to the first round (metadata chain, first batch) */
#endif
    for (;;) {
        const uint32_t qmin = __reduce_min_sync(FULL, done ? 0xffffffffu : qp);
        if (qmin == 0xffffffffu) break; /* every lane is finished */
        const uint32_t f = qmin < 32 ? 0u : (qmin - 32) >> 5; /* rows below f are dead (q may step back by < 32 bits when a window changes) */
#pragma unroll 1
        while (issued_b < total_b && (issued_b + 1) * B <= f + NW) { issue(issued_b); issued_b++; }
        /* the rows the lanes may touch this round must have landed; batches beyond the most advanced lane's look-ahead stay in
         * flight (they were issued when the ring had room, about two rounds before they are needed) */
        const uint32_t qmax = __reduce_max_sync(FULL, done ? 0u : qp);
        uint32_t need_max = ((qmax + OG_IL_LOOKBITS) >> 5) + 1; if (need_max > rows_w) need_max = rows_w;
        uint32_t want_b = (need_max + B - 1) / B; if (want_b > issued_b) want_b = issued_b;
#ifdef OG_IL_STATS
        st_w0 = clock64();
#endif
#pragma unroll 1
        while (ready_b < want_b) { if (!mbar_wait(bar0 + (ready_b % NB) * 8, (ready_b / NB) & 1)) { hung = 1; break; } ready_b++; }
#ifdef OG_IL_STATS
        st_wait += clock64() - st_w0;
#endif
        if (hung) break;
        uint32_t need = ((qp + OG_IL_LOOKBITS) >> 5) + 1; if (need > rows_w) need = rows_w;
        bool go = done || need <= ready_b * B; /* a lane that could touch rows not resident yet sits the round out */
        uint32_t run = __reduce_min_sync(FULL, go ? n_ev : 0u); /* finished lanes have n_ev near 2^32 */
        if (run >= K) { /* every lane runs, no boundary ahead */
            static_assert(K % 2 == 0, "records are decoded in pairs");
#pragma unroll UNR
            for (uint32_t k = 0; k < K; k += 2) record2(k);
            n_ev -= K;
#ifdef OG_IL_STATS
            st_common++;
#endif
            continue;
        }
#ifdef OG_IL_STATS
        st_rare++;
#endif
        /* ---- the rare round ---- */
        if (rounds_left-- == 0) { hung = 2; break; }
        const bool all_go = __all_sync(FULL, go); /* false: some lane is so far ahead of the slowest one that the ring cannot hold both */
#ifdef OG_IL_STATS
        if (!all_go) { st_notgo++; st_sit += __popc(__ballot_sync(FULL, !go)); }
#endif
        /* K records per running lane, in runs that end where the first lane reaches a window boundary */
        uint32_t left = K;
        for (;;) {
            run = __reduce_min_sync(FULL, go ? n_ev : 0xffffffffu);
            if (run > left) run = left;
            if (all_go) {
#pragma unroll 1
                for (uint32_t k = 0; k < run; k++) record(k);
            } else {
#pragma unroll 1
                for (uint32_t k = 0; k < run; k++) if (go) record(k);
            }
            if (go) n_ev -= run;
            left -= run;
            if (left == 0) break;
            const bool ev = go && !done && n_ev == 0; /* current row == stop */
            if (FOLD && uni) {
                const bool fl = ev && !skipping;
                const int kind = kind_of();
                const bool to_acc = fl && (kind == 2 || fold_edges);
                if (fl && !to_acc) flush_lane(kind);
                if (__any_sync(FULL, to_acc)) flush_fold(to_acc);
                if (to_acc && kind == 0) head_done = true;
            } else if (ev && !skipping) flush_lane(kind_of());
            if (ev) advance();
            /* every live lane crossed a window boundary in the same step (lanes that share a time grid always do): start a fresh
             * round here, so that the rest of this window runs in common rounds instead of finishing this round record by record.
             * Windows then stay aligned to rounds (60-row windows = 5 rounds of 12) */
            if (__all_sync(FULL, ev || done)) break;
        }
    }
    if (active && (qp >> 5) >= rows_w) bad = 1; /* ran past the stream: corrupt page */
#ifdef OG_IL_STATS
    const long long st_e0 = clock64(); /* epilogue: last round to warp end (drain, cell and edge stores) */
    if (lane == 0) { atomicAdd((unsigned *)&ch.err[4], st_common); atomicAdd((unsigned *)&ch.err[5], st_rare); atomicAdd((unsigned *)&ch.err[6], st_notgo); atomicAdd((unsigned *)&ch.err[7], st_sit); }
#endif
    /* copies still in flight must land before this CTA's shared memory can be reused */
    while (ready_b < issued_b && hung != 1) { if (!mbar_wait(bar0 + (ready_b % NB) * 8, (ready_b / NB) & 1)) hung = 1; ready_b++; }
    if (hung && lane == 0) report_err(ch.err, D_WATCHDOG, (grp << 2) | hung);
    if (FOLD && uni) { /* the group's folded windows -> one cell per bucket (the tail window to the tail column) */
        __syncwarp();
        const uint32_t w_tail = fold_edges ? b_end - b0 : OG_IL_WCAP;
        for (uint32_t i = lane; i < OG_IL_WCAP * q.n_calls; i += 32) {
            if (!acc_k[i]) continue;
            const uint32_t c = i / OG_IL_WCAP, w = i % OG_IL_WCAP;
            Part a; a.ok = 1; a.v = acc_v[i]; a.t = TIMES ? acc_t[i] : 0;
            store_part(ch.gcells[c], (size_t)(b0 + w) * ch.gc_cols + (w == w_tail ? ch.gc_tail0 + gcol : gcol), a);
        }
    }
    /* some lane wrote edge windows: k_fix_edges_fold has work */
    if (FOLD && __any_sync(FULL, active && head_b != OG_NO_BUCKET) && lane == 0) ch.flags[1] = 1;
    if (active) {
        if (bad) report_err(ch.err, D_CORRUPT, seg);
        *(uint2 *)(ch.edge_bucket + e) = make_uint2(head_b, (head_b == OG_NO_BUCKET || cur_b == head_b) ? OG_NO_BUCKET : cur_b);
    }
#ifdef OG_IL_STATS
    if (lane == 0) {
        atomicAdd((unsigned long long *)(ch.err + 8), (unsigned long long)st_wait);
        const long long st_end = clock64();
        atomicAdd((unsigned long long *)(ch.err + 10), (unsigned long long)(st_end - st_clk0));
        atomicAdd((unsigned long long *)(ch.err + 12), (unsigned long long)st_pro);
        atomicAdd((unsigned long long *)(ch.err + 14), (unsigned long long)(st_end - st_e0));
    }
#endif
}

} // namespace ogpu
