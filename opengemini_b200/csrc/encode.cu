/*
 * encode.cu — K7: page encoders on the device, and the synthetic shard generator that uses them.
 *
 * One thread encodes one segment page (codec selection needs whole-segment statistics and the bit streams are
 * serial).  Reference functions replaced:
 *   encode_float_page  ColumnBuilder.encFloatColumn column_builder.go:201 -> EncodeColumnHeader :428 ->
 *                      compress.Float.adaptiveEncoding lib/compress/float.go:60-101 (GenerateContext :210) ->
 *                      tsm1.FloatArrayEncodeAll batch_float.go:17 | RLE.Encoding compress.go:68 | SameValueEncoding :38
 *   encode_int_page    encIntegerColumn :151 -> Integer.Encoding lib/encoding/int.go:183 (const-delta :101, simple8b :123,
 *                      raw :168; simple8b.EncodeAll simple8b/encoding.go:350)
 *   encode_time_page   ChunkDataBuilder.EncodeTime chunkdata_builder.go:65 -> Time.Encoding timestamp.go:150
 *   encode_bool_page   encBooleanColumn :299 -> Boolean.Encoding bool.go:40
 * Deviations (documented in DESIGN.md): where the reference would call a third-party compressor (Snappy for
 * "few-decimal"/NaN floats and irregular timestamps, zstd for ints with >60-bit deltas) this encoder writes the
 * uncompressed form of the same block (float tag 0, time tag 4, int tag 4) — still a valid page for the Go reader.
 */
#include <algorithm>
#include <cstdio>
#include <cstring>

#include "../../include/ogpu_synth.h"
#include "decode.cuh"
#include "internal.h"

namespace ogpu {

#define PAGE_STRIDE 8704u /* staging bytes per page: worst case 13 + 125 + 1 + 8000 (raw) rounded up, 8-byte aligned */

/* MSB-first bit writer with 8-byte aligned big-endian stores */
struct BitWriter {
    uint8_t *out; uint64_t acc; unsigned nacc; uint32_t nbytes;
    __device__ __forceinline__ void init(uint8_t *o) { out = o; acc = 0; nacc = 0; nbytes = 0; }
    __device__ __forceinline__ void flush8() { *(uint64_t *)(out + nbytes) = bswap64(acc); nbytes += 8; acc = 0; nacc = 0; }
    __device__ __forceinline__ void put(uint64_t v, unsigned k) { /* low k bits of v, 1 <= k <= 64 */
        if (k < 64) v &= (1ull << k) - 1;
        unsigned room = 64 - nacc;
        if (k <= room) { acc |= (k == 64) ? v : (v << (room - k)); nacc += k; if (nacc == 64) flush8(); }
        else { unsigned rest = k - room; acc |= v >> rest; flush8(); acc = v << (64 - rest); nacc = rest; }
    }
    __device__ __forceinline__ void put_bytes_le64(uint64_t v) { put(bswap64(v), 64); } /* raw little-endian 8 bytes */
    __device__ __forceinline__ uint32_t finish() { /* pad to a byte, flush, return total length */
        uint32_t total = nbytes + (nacc + 7) / 8;
        if (nacc) { *(uint64_t *)(out + nbytes) = bswap64(acc); }
        return total;
    }
    __device__ __forceinline__ uint32_t bits() const { return nbytes * 8 + nacc; }
};

__device__ __forceinline__ void put_uvarint(BitWriter &w, uint64_t v) {
    while (v >= 0x80) { w.put((v & 0x7f) | 0x80, 8); v >>= 7; }
    w.put(v, 8);
}
__device__ __forceinline__ uint64_t zigzag_enc(int64_t v) { return ((uint64_t)v << 1) ^ (uint64_t)(v >> 63); }

/* segment view handed to the encoders: one 8-byte (bool: 1-byte) cell per ROW plus an optional validity byte per row */
struct SegIn {
    const uint8_t *cells; const uint8_t *okb; uint32_t rows; int wide;
    __device__ __forceinline__ bool valid(uint32_t r) const { return !okb || okb[r]; }
    __device__ __forceinline__ uint64_t cell(uint32_t r) const { return wide ? ((const uint64_t *)cells)[r] : (uint64_t)cells[r]; }
};

/* EncodeColumnHeader column_builder.go:428-444; returns non-null count */
__device__ uint32_t write_header(BitWriter &w, const SegIn &s, int type) {
    uint32_t n = 0;
    for (uint32_t r = 0; r < s.rows; r++) n += s.valid(r) ? 1u : 0u;
    uint32_t nil = s.rows - n;
    uint8_t full = type == OG_TYPE_FLOAT ? 31 : type == OG_TYPE_INT ? 32 : 33;
    if (nil == 0) { w.put(full, 8); w.put(s.rows, 32); return n; }
    if (nil == s.rows) { w.put(full + 10, 8); w.put(s.rows, 32); return n; }
    w.put((uint64_t)type, 8);
    uint32_t nb = (s.rows + 7) / 8;
    w.put(nb, 32);
    for (uint32_t i = 0; i < nb; i++) {
        uint32_t v = 0;
        for (uint32_t k = 0; k < 8 && i * 8 + k < s.rows; k++) v |= (s.valid(i * 8 + k) ? 1u : 0u) << k;
        w.put(v, 8);
    }
    w.put(0, 32);   /* bitmap offset */
    w.put(nil, 32); /* NullN */
    return n;
}

/* ---- float: adaptive selection ---- */
__device__ __forceinline__ bool is_int_f(double f) { /* isInt float.go:240-246 */
    if (f >= 0 && f < 4294967296.0) return (double)(unsigned long long)f == f;
    return ceil(f) == f && floor(f) == f;
}

/* returns false when the stream grew past limit_bytes (the caller falls back to the raw block, exactly what the
 * reference does after finishing the encode: float.go:96-99) */
__device__ bool gorilla_encode_dev(BitWriter &w, const SegIn &s, uint32_t limit_bytes) { /* FloatArrayEncodeAll batch_float.go:17-254 */
    w.put(0x10, 8);
    uint32_t r = 0;
    while (!s.valid(r)) r++;
    uint64_t prev = s.cell(r); r++;
    w.put(prev, 64);
    uint64_t prev_leading = ~0ull, prev_trailing = 0;
    bool finished = false;
    while (!finished) {
        if (w.nbytes > limit_bytes) return false;
        uint64_t cur;
        while (r < s.rows && !s.valid(r)) r++;
        if (r < s.rows) { cur = s.cell(r); r++; }
        else { cur = OG_UVNAN; finished = true; }
        uint64_t delta = cur ^ prev;
        if (delta == 0) { w.put(0, 1); prev = cur; continue; }
        uint64_t leading = (uint64_t)__clzll((long long)delta) & 0x1F; /* :88-91 */
        uint64_t trailing = (uint64_t)(__ffsll((long long)delta) - 1);
        if (prev_leading != ~0ull && leading >= prev_leading && trailing >= prev_trailing) {
            w.put(2, 2); /* '1','0' */
            w.put(delta >> prev_trailing, (unsigned)(64 - prev_leading - prev_trailing));
        } else {
            prev_leading = leading; prev_trailing = trailing;
            uint64_t sig = 64 - leading - trailing;
            w.put((3ull << 11) | (leading << 6) | (sig & 0x3F), 13); /* '1','1', 5 bits leading, 6 bits sigbits */
            w.put(delta >> trailing, (unsigned)sig);
        }
        prev = cur;
    }
    return true;
}

/* nan_raw: a segment that FloatArrayEncodeAll refuses (sum over src[1:] is NaN: +Inf and -Inf in one segment) gets the raw
 * block instead of flag 2 (the open-time merge re-encodes rows it must not drop, merge.cu) */
__device__ uint32_t encode_float_page(uint8_t *out, const SegIn &s, int *flags, bool nan_raw) {
    BitWriter w; w.init(out);
    if (s.rows == 1 && s.valid(0)) { w.put(17, 8); w.put_bytes_le64(s.cell(0)); return w.finish(); } /* CanEncodeOneRowMode :488 */
    uint32_t n = write_header(w, s, OG_TYPE_FLOAT);
    if (n == 0) return w.finish();
    /* GenerateContext float.go:210-238 */
    uint32_t distinct = 1; bool extreme = false, int_only = true, less_dec = true;
    double sum_tail = 0; /* FloatArrayEncodeAll's running sum over src[1:] (batch_float.go:55,245) */
    if (n > 4) {
        uint64_t pv = 0; bool have = false;
        for (uint32_t r = 0; r < s.rows; r++) {
            if (!s.valid(r)) continue;
            uint64_t u = s.cell(r); double d = __longlong_as_double((long long)u);
            if (have) sum_tail += d;
            if (have && d != __longlong_as_double((long long)pv)) distinct++;
            if (d != d) extreme = true;
            pv = u; have = true;
        }
        if (distinct > 8) {
            uint32_t k = 0, less_total = 0, i = 0;
            for (uint32_t r = 0; r < s.rows && i < n && k < n / 10; r++) {
                if (!s.valid(r)) continue;
                i++;
                double d = __longlong_as_double((long long)s.cell(r));
                if (d == 0) continue;
                k++;
                if (int_only && !is_int_f(d)) int_only = false;
                if (is_int_f(__dmul_rn(d, 1000.0))) less_total++;
            }
            less_dec = k > 0 && (100 * less_total / k) > 90;
        }
    }
    uint32_t hdr_bits = w.bits();
    auto raw = [&]() { /* compressNull :133-137 */
        w.put(0x00, 8);
        for (uint32_t r = 0; r < s.rows; r++) if (s.valid(r)) w.put_bytes_le64(s.cell(r));
    };
    if (n <= 4) { raw(); return w.finish(); }
    if (distinct == 1) { /* SameValueEncoding compress.go:38-49 */
        w.put(0x40, 8); w.put(n & 0xffff, 16);
        uint32_t r = 0; while (!s.valid(r)) r++;
        uint64_t u = s.cell(r);
        if (__longlong_as_double((long long)u) != 0) w.put_bytes_le64(u);
        return w.finish();
    }
    if (distinct <= 8) { /* RLE.Encoding compress.go:68-93 (bit-pattern equality, 16384 cap) */
        w.put(0x50, 8);
        uint64_t run_v = 0; uint32_t run = 0;
        auto emit = [&]() {
            if (run_v == 0) w.put(run | (1u << 15), 16);
            else { w.put(run, 16); w.put_bytes_le64(run_v); }
        };
        for (uint32_t r = 0; r < s.rows; r++) {
            if (!s.valid(r)) continue;
            uint64_t u = s.cell(r);
            if (run && u == run_v && run < (1u << 14)) { run++; continue; }
            if (run) emit();
            run_v = u; run = 1;
        }
        emit();
        return w.finish();
    }
    if ((!int_only && less_dec) || extreme) { /* reference: Snappy (third-party). device: raw block, flagged */
        if (flags) atomicOr(flags, 1);
        raw(); return w.finish();
    }
    if (sum_tail != sum_tail) { /* "unsupported value: NaN" (+Inf and -Inf in one segment) */
        if (nan_raw) { raw(); return w.finish(); }
        if (flags) atomicOr(flags, 2);
    }
    w.put(0x30, 8);
    uint32_t limit = n * 8 * 90 / 100;
    bool fits = gorilla_encode_dev(w, s, hdr_bits / 8 + limit + 16);
    uint32_t total = w.finish();
    uint32_t block = total - hdr_bits / 8;
    if (!fits || block > limit) { /* float.go:96-99 */
        w.init(out);
        write_header(w, s, OG_TYPE_FLOAT);
        raw();
        return w.finish();
    }
    return total;
}

/* ---- simple8b greedy packer over a random-access source (simple8b.EncodeAll :350 incl. the canPack quirk :455-462) ---- */
template <class Src>
__device__ void s8b_pack(BitWriter &w, Src src, uint32_t n, uint32_t *n_words, bool count_only) {
    const unsigned N[16] = {240, 120, 60, 30, 20, 15, 12, 10, 8, 7, 6, 5, 4, 3, 2, 1};
    const unsigned B[16] = {0, 0, 1, 2, 3, 4, 5, 6, 7, 8, 10, 12, 15, 20, 30, 60};
    int last_non_one = -1;
    for (uint32_t i = 0; i < n; i++) if (src(i) != 1) last_non_one = (int)i;
    uint32_t i = 0, words = 0;
    while (i < n) {
        uint32_t rem = n - i;
        unsigned sel;
        bool all_one = (int)i > last_non_one;
        if (rem >= 240 && all_one) sel = 0;
        else if (rem >= 120 && all_one) sel = 1;
        else {
            unsigned need = 0, lim = rem < 60 ? rem : 60;
            unsigned need_at[61];
            for (unsigned k = 0; k < lim; k++) { uint64_t v = src(i + k); unsigned b = v ? 64 - (unsigned)__clzll((long long)v) : 0; if (b > need) need = b; need_at[k + 1] = need; }
            sel = 15;
            for (unsigned sI = 2; sI < 16; sI++) if (rem >= N[sI] && need_at[N[sI]] <= B[sI]) { sel = sI; break; }
        }
        if (!count_only) {
            uint64_t word = (uint64_t)sel << 60;
            if (sel >= 2) for (unsigned k = 0; k < N[sel]; k++) word |= src(i + k) << (k * B[sel]);
            w.put(word, 64);
        }
        i += N[sel]; words++;
    }
    *n_words = words;
}

__device__ uint32_t encode_int_page(uint8_t *out, const SegIn &s, int *flags) {
    BitWriter w; w.init(out);
    if (s.rows == 1 && s.valid(0)) { w.put(18, 8); w.put_bytes_le64(s.cell(0)); return w.finish(); }
    uint32_t n = write_header(w, s, OG_TYPE_INT);
    if (n == 0) return w.finish();
    /* the non-null values are read through a compacting index: nulls are rare, so a forward scan per access is avoided by
       requiring the caller to pass dense cells when nulls exist (see k_encode_pages: compaction into scratch) */
    const int64_t *v = (const int64_t *)s.cells;
    auto raw = [&]() { w.put(0x40, 8); w.put(n * 8, 32); for (uint32_t i = 0; i < n; i++) w.put(zigzag_enc(v[i]), 64); };
    if (n < 3) { raw(); return w.finish(); }
    bool is_const = true, is_s8b = true;
    uint64_t d1 = zigzag_enc((int64_t)((uint64_t)v[1] - (uint64_t)v[0]));
    if (d1 > ((1ull << 60) - 1)) is_s8b = false;
    uint64_t pd = d1;
    for (uint32_t i = 2; i < n; i++) {
        uint64_t e = zigzag_enc((int64_t)((uint64_t)v[i] - (uint64_t)v[i - 1]));
        is_const = is_const && pd == e;
        if (e > ((1ull << 60) - 1)) is_s8b = false;
        pd = e;
    }
    if (is_const) { w.put(0x10, 8); w.put(zigzag_enc(v[0]), 64); put_uvarint(w, d1); put_uvarint(w, (uint64_t)n - 1); return w.finish(); }
    if (is_s8b) {
        auto src = [&](uint32_t i) { return zigzag_enc((int64_t)((uint64_t)v[i + 1] - (uint64_t)v[i])); };
        uint32_t words = 0;
        s8b_pack(w, src, n - 1, &words, true);
        w.put(0x20, 8); w.put(words + 1, 32); w.put(n, 32); w.put(zigzag_enc(v[0]), 64);
        s8b_pack(w, src, n - 1, &words, false);
        return w.finish();
    }
    if (flags) atomicOr(flags, 4); /* reference: zstd */
    raw();
    return w.finish();
}

__device__ uint32_t encode_time_page(uint8_t *out, const int64_t *tv, uint32_t n, int *flags) {
    BitWriter w; w.init(out);
    if (n == 1) { w.put(18, 8); w.put_bytes_le64((uint64_t)tv[0]); return w.finish(); }
    w.put(32, 8); w.put(n, 32);
    const uint64_t *t = (const uint64_t *)tv;
    auto raw = [&]() { w.put(0x40, 8); w.put(n * 8, 32); for (uint32_t i = 0; i < n; i++) w.put(zigzag_enc(tv[i]), 64); };
    if (n < 3) { raw(); return w.finish(); }
    /* encodingInit timestamp.go:63-83 */
    const uint64_t SC[12] = {10ull, 100ull, 1000ull, 10000ull, 100000ull, 1000000ull, 10000000ull, 100000000ull, 1000000000ull, 10000000000ull, 100000000000ull, 1000000000000ull};
    uint64_t dl = t[n - 1] - t[n - 2];
    bool is_const = true, is_s8b = dl < ((1ull << 60) - 1);
    uint64_t sc = 1;
    for (int i = 11; i > 0; i--) if (dl % SC[i] == 0) { sc = SC[i]; break; }
    uint64_t nd = dl;
    for (uint32_t i = n - 2; i > 0; i--) {
        uint64_t d = t[i] - t[i - 1];
        while (sc > 1 && d % sc != 0) sc /= 10;
        is_const = is_const && d == nd;
        is_s8b = is_s8b && d < ((1ull << 60) - 1);
        nd = d;
    }
    if (is_const) { w.put(0x10, 8); w.put(t[0], 64); put_uvarint(w, t[1] - t[0]); put_uvarint(w, (uint64_t)n - 1); return w.finish(); }
    if (is_s8b) {
        auto src = [&](uint32_t i) { return (t[i + 1] - t[i]) / sc; };
        uint32_t words = 0;
        s8b_pack(w, src, n - 1, &words, true);
        w.put(0x20, 8); w.put(sc, 64); w.put(words + 1, 32); w.put(n, 32); w.put(t[0], 64);
        s8b_pack(w, src, n - 1, &words, false);
        return w.finish();
    }
    if (flags) atomicOr(flags, 8); /* reference: snappy */
    raw();
    return w.finish();
}

__device__ uint32_t encode_bool_page(uint8_t *out, const SegIn &s) {
    BitWriter w; w.init(out);
    if (s.rows == 1 && s.valid(0)) { w.put(19, 8); w.put(s.cell(0) ? 1 : 0, 8); return w.finish(); }
    uint32_t n = write_header(w, s, OG_TYPE_BOOL);
    if (n == 0) return w.finish();
    w.put(0x10, 8); w.put(n, 32);
    for (uint32_t r = 0; r < s.rows; r++) if (s.valid(r)) w.put(s.cell(r) ? 1 : 0, 1);
    return w.finish(); /* Flush(Zero): zero padding to the byte */
}

/* one thread per segment: encode into staging[seg * PAGE_STRIDE], record the length */
__global__ void k_encode_pages(int type, int is_time, const uint8_t *cells, const uint8_t *okb, const uint32_t *rows_arr,
                               uint32_t n_segments, uint32_t rps, uint8_t *staging, uint32_t *lens, uint64_t *dense_scratch, int *flags,
                               bool nan_raw) {
    uint32_t seg = blockIdx.x * blockDim.x + threadIdx.x;
    if (seg >= n_segments) return;
    uint32_t rows = rows_arr ? rows_arr[seg] : rps;
    uint8_t *out = staging + (size_t)seg * PAGE_STRIDE;
    int wide = type != OG_TYPE_BOOL;
    SegIn s; s.rows = rows; s.wide = wide;
    s.cells = cells + (size_t)seg * rps * (wide ? 8 : 1);
    s.okb = okb ? okb + (size_t)seg * rps : nullptr;
    uint32_t len;
    if (is_time) len = encode_time_page(out, (const int64_t *)s.cells, rows, flags);
    else if (type == OG_TYPE_FLOAT) len = encode_float_page(out, s, flags, nan_raw);
    else if (type == OG_TYPE_BOOL) len = encode_bool_page(out, s);
    else {
        if (s.okb) { /* compact the non-null ints so the delta logic sees ColVal.Val */
            uint64_t *ds = dense_scratch + (size_t)seg * rps; uint32_t k = 0;
            for (uint32_t r = 0; r < rows; r++) if (s.okb[r]) ds[k++] = ((const uint64_t *)s.cells)[r];
            /* encode_int_page reads values as dense ColVal.Val: hand it the compacted copy, keep okb for the header */
            SegIn d2; d2.rows = rows; d2.wide = 1; d2.okb = s.okb; d2.cells = (const uint8_t *)ds;
            len = encode_int_page(out, d2, flags);
        } else len = encode_int_page(out, s, flags);
    }
    lens[seg] = len;
}

/* exclusive scan of page lengths: single block, good for <= a few hundred thousand pages per batch */
__global__ void k_scan_lens(const uint32_t *lens, uint32_t n, uint64_t base, uint64_t *offs, unsigned long long *total) {
    __shared__ unsigned long long part[1024];
    uint32_t per = (n + blockDim.x - 1) / blockDim.x;
    uint32_t a = threadIdx.x * per, b = min(n, a + per);
    unsigned long long sum = 0;
    for (uint32_t i = a; i < b; i++) sum += lens[i];
    part[threadIdx.x] = sum;
    __syncthreads();
    if (threadIdx.x == 0) { unsigned long long run = 0; for (uint32_t i = 0; i < blockDim.x; i++) { unsigned long long v = part[i]; part[i] = run; run += v; } *total = run; }
    __syncthreads();
    unsigned long long run = part[threadIdx.x] + base;
    for (uint32_t i = a; i < b; i++) { offs[i] = run; run += lens[i]; }
}

/* one warp per page: copy staging -> packed blob */
__global__ void k_compact_pages(const uint8_t *staging, const uint32_t *lens, const uint64_t *offs, uint32_t n, uint8_t *blob, uint64_t cap, int *flags) {
    uint32_t page = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (page >= n) return;
    uint32_t len = lens[page]; uint64_t off = offs[page];
    if (off + len > cap) { if (lane == 0) atomicOr(flags, 16); return; }
    const uint8_t *src = staging + (size_t)page * PAGE_STRIDE;
    uint8_t *dst = blob + off;
    for (uint32_t i = lane; i < len; i += 32) dst[i] = src[i];
}

/* synthetic rows for a batch of segments of one column (include/ogpu_synth.h) */
__global__ void k_synth_fill(og_synth_desc d, og_synth_column col, uint32_t column, uint32_t seg_begin, uint32_t n_segments,
                             uint32_t segs_per_series, uint8_t *cells, uint8_t *okb) {
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_segments) return;
    uint32_t seg = seg_begin + i, series = d.series_base + seg / segs_per_series, g = seg % segs_per_series;
    uint32_t rps = d.rows_per_segment;
    uint64_t row0 = (uint64_t)g * rps;
    uint32_t n = (uint32_t)min((uint64_t)rps, (uint64_t)d.rows_per_series - row0);
    int wide = col.type != OG_TYPE_BOOL;
    uint8_t *c = cells + (size_t)i * rps * (wide ? 8 : 1);
    uint8_t *ok = okb ? okb + (size_t)i * rps : nullptr;
    int64_t walk = 0;
    for (uint32_t k = 0; k < n; k++) {
        uint64_t row = row0 + k;
        uint64_t bits;
        switch (col.dist) {
        case OG_SYNTH_F_HI: bits = (uint64_t)__double_as_longlong(og_synth_f_hi(d.seed, column, series, row)); break;
        case OG_SYNTH_F_LO:
            walk = k == 0 ? og_synth_walk_first(d.seed, column, series, g, 1) : walk + og_synth_f_lo_step(d.seed, column, series, row);
            bits = (uint64_t)__double_as_longlong((double)walk); break;
        case OG_SYNTH_INT_WALK:
            walk = k == 0 ? og_synth_walk_first(d.seed, column, series, g, 0) : walk + og_synth_int_step(d.seed, column, series, row);
            bits = (uint64_t)walk; break;
        default: bits = (uint64_t)og_synth_bool(d.seed, column, series, row); break;
        }
        if (wide) ((uint64_t *)c)[k] = bits; else c[k] = (uint8_t)bits;
        if (ok) ok[k] = og_synth_is_null(d.seed, column, series, row, col.null_permille) ? 0 : 1;
    }
}

__global__ void k_synth_times(og_synth_desc d, uint32_t seg_begin, uint32_t n_segments, uint32_t segs_per_series, int64_t *cells,
                              uint32_t *rows_arr, int64_t *tmin, int64_t *tmax) {
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_segments) return;
    uint32_t seg = seg_begin + i, g = seg % segs_per_series;
    uint32_t rps = d.rows_per_segment;
    uint64_t row0 = (uint64_t)g * rps;
    uint32_t n = (uint32_t)min((uint64_t)rps, (uint64_t)d.rows_per_series - row0);
    int64_t *c = cells + (size_t)i * rps;
    for (uint32_t k = 0; k < n; k++) c[k] = d.t0 + (int64_t)(row0 + k) * d.dt;
    rows_arr[i] = n;
    tmin[seg] = c[0]; tmax[seg] = c[n - 1];
}

} // namespace ogpu

using namespace ogpu;

extern "C" {

} // extern "C"
namespace ogpu {
/* og_encode_pages; nan_raw: see encode_float_page */
int encode_pages(int32_t type, int32_t is_time, const void *d_values, const uint8_t *d_valid, const uint32_t *d_rows, uint32_t n_segments,
                 uint32_t rps, uint8_t *d_out, uint64_t out_cap, uint64_t *d_page_off, uint32_t *d_page_len, uint64_t *total_bytes_out, bool nan_raw) {
    if (!d_values || !d_out || !d_page_off || !d_page_len || rps == 0 || rps > 1000) { set_error("bad argument (rows_per_segment must be 1..1000)"); return OG_E_INVAL; }
    if (type != OG_TYPE_INT && type != OG_TYPE_FLOAT && type != OG_TYPE_BOOL) { set_error("unsupported column type %d", type); return OG_E_UNSUPPORTED; }
    if (n_segments == 0) { if (total_bytes_out) *total_bytes_out = 0; return OG_OK; }
    { int rcd = ensure_device(); if (rcd) return rcd; }
    Scratch tmp;
    uint8_t *staging; uint64_t *dense = nullptr; int *flags; unsigned long long *d_total;
    int rc;
    if ((rc = tmp.get(&staging, (size_t)n_segments * PAGE_STRIDE))) return rc;
    if (type == OG_TYPE_INT && d_valid && !is_time && (rc = tmp.get(&dense, (size_t)n_segments * rps))) return rc;
    if ((rc = tmp.get(&flags, 1)) || (rc = tmp.get(&d_total, 1))) return rc;
    cudaMemset(flags, 0, 4);
    k_encode_pages<<<(n_segments + 63) / 64, 64>>>(type, is_time, (const uint8_t *)d_values, is_time ? nullptr : d_valid, d_rows, n_segments, rps, staging, d_page_len, dense, flags, nan_raw);
    k_scan_lens<<<1, 1024>>>(d_page_len, n_segments, 0, d_page_off, d_total);
    k_compact_pages<<<(unsigned)(((size_t)n_segments * 32 + 255) / 256), 256>>>(staging, d_page_len, d_page_off, n_segments, d_out, out_cap, flags);
    unsigned long long total = 0; int fl = 0;
    cudaError_t e = cudaMemcpy(&total, d_total, 8, cudaMemcpyDeviceToHost);
    if (e == cudaSuccess) e = cudaMemcpy(&fl, flags, 4, cudaMemcpyDeviceToHost);
    if (e != cudaSuccess) return cuda_fail(e, "og_encode_pages", __FILE__, __LINE__);
    if (fl & 2) { set_error("float column contains +Inf and -Inf (or NaN): FloatArrayEncodeAll rejects it (batch_float.go:245)"); return OG_E_INVAL; }
    if (fl & 16) { set_error("output buffer too small (%llu bytes needed)", total); return OG_E_NOMEM; }
    if (total_bytes_out) *total_bytes_out = total;
    return OG_OK;
}
} // namespace ogpu
extern "C" {

OG_API int og_encode_pages(int32_t type, int32_t is_time, const void *d_values, const uint8_t *d_valid, const uint32_t *d_rows,
                           uint32_t n_segments, uint32_t rps, uint8_t *d_out, uint64_t out_cap, uint64_t *d_page_off,
                           uint32_t *d_page_len, uint64_t *total_bytes_out) {
    return encode_pages(type, is_time, d_values, d_valid, d_rows, n_segments, rps, d_out, out_cap, d_page_off, d_page_len, total_bytes_out, false);
}

OG_API int og_shard_synth(const og_synth_desc *dd, og_shard **out) {
    if (!dd || !out || dd->n_series == 0 || dd->rows_per_series == 0 || dd->n_columns == 0 || dd->n_columns > 8) { set_error("bad synth descriptor"); return OG_E_INVAL; }
    *out = nullptr;
    og_synth_desc d = *dd;
    if (d.rows_per_segment == 0) d.rows_per_segment = 1000;
    if (d.rows_per_segment > 1000 || d.dt <= 0) { set_error("rows_per_segment must be <= 1000 and dt > 0"); return OG_E_INVAL; }
    { int rcd = ensure_device(); if (rcd) return rcd; }
    int dev = 0; if (cudaGetDevice(&dev) != cudaSuccess) return OG_E_CUDA;
    uint32_t rps = d.rows_per_segment;
    uint32_t sps = (d.rows_per_series + rps - 1) / rps;
    uint64_t nseg64 = (uint64_t)d.n_series * sps;
    if (nseg64 > 0xfffffff0ull) { set_error("too many segments"); return OG_E_INVAL; }
    uint32_t nseg = (uint32_t)nseg64;
    std::unique_ptr<og_shard> s(new og_shard);
    s->device = dev; s->n_series = d.n_series; s->n_segments = nseg; s->n_columns = d.n_columns;
    for (uint32_t c = 0; c < d.n_columns; c++) { s->col_types.push_back(d.columns[c].type); s->col_names.push_back("f" + std::to_string(c)); }
    s->sids.resize(d.n_series); s->h_series_seg_begin.resize((size_t)d.n_series + 1);
    for (uint32_t i = 0; i < d.n_series; i++) { s->sids[i] = (uint64_t)d.series_base + i + 1; s->h_series_seg_begin[i] = i * sps; }
    s->h_series_seg_begin[d.n_series] = nseg;
    s->tmin = d.t0; s->tmax = d.t0 + (int64_t)(d.rows_per_series - 1) * d.dt;
    int rc;
    size_t ncol1 = (size_t)d.n_columns + 1;
    if ((rc = alloc_dir(s.get()))) return rc; /* seg_tmin / seg_tmax and the page directory are filled on the device */
    CU(cudaMemcpy(s->d_series_seg_begin, s->h_series_seg_begin.data(), ((size_t)d.n_series + 1) * 4, cudaMemcpyHostToDevice));
    CU(cudaMemcpy(s->d_sids, s->sids.data(), (size_t)d.n_series * 8, cudaMemcpyHostToDevice));
    /* batch scratch */
    uint32_t batch = std::min<uint32_t>(nseg, 128u * 1024u);
    uint8_t *cells, *okb, *staging; uint32_t *rows_arr, *lens; uint64_t *offs, *dense; int *flags; unsigned long long *d_total;
    Scratch tmp;
    if ((rc = tmp.get(&cells, (size_t)batch * rps * 8)) || (rc = tmp.get(&okb, (size_t)batch * rps)) || (rc = tmp.get(&staging, (size_t)batch * PAGE_STRIDE)) ||
        (rc = tmp.get(&rows_arr, batch)) || (rc = tmp.get(&lens, batch)) || (rc = tmp.get(&offs, batch)) || (rc = tmp.get(&dense, (size_t)batch * rps)) ||
        (rc = tmp.get(&flags, 1)) || (rc = tmp.get(&d_total, 1)))
        return rc;
    CU(cudaMemset(flags, 0, 4));
    /* pass 0: size estimate from the first batch of every column, then allocate the blob once */
    std::vector<double> avg(ncol1, 0);
    auto run_batch = [&](uint32_t c, uint32_t b0, uint32_t n, uint8_t *blob, uint64_t base, uint64_t cap, unsigned long long *tot) -> int {
        unsigned g = (n + 127) / 128;
        if (c == d.n_columns) {
            k_synth_times<<<g, 128>>>(d, b0, n, sps, (int64_t *)cells, rows_arr, s->d_tmin, s->d_tmax);
            k_encode_pages<<<(n + 63) / 64, 64>>>(OG_TYPE_INT, 1, cells, nullptr, rows_arr, n, rps, staging, lens, nullptr, flags, false);
        } else {
            const og_synth_column &col = d.columns[c];
            k_synth_times<<<g, 128>>>(d, b0, n, sps, (int64_t *)cells, rows_arr, s->d_tmin, s->d_tmax); /* rows_arr (overwritten cells are refilled below) */
            k_synth_fill<<<g, 128>>>(d, col, c, b0, n, sps, cells, col.null_permille ? okb : nullptr);
            k_encode_pages<<<(n + 63) / 64, 64>>>(col.type, 0, cells, col.null_permille ? okb : nullptr, rows_arr, n, rps, staging, lens, dense, flags, false);
        }
        k_scan_lens<<<1, 1024>>>(lens, n, base, offs, d_total);
        if (blob) {
            k_compact_pages<<<(unsigned)(((size_t)n * 32 + 255) / 256), 256>>>(staging, lens, offs, n, blob, cap, flags);
            cudaMemcpyAsync(s->d_page_off + (size_t)c * nseg + b0, offs, (size_t)n * 8, cudaMemcpyDeviceToDevice);
            cudaMemcpyAsync(s->d_page_len + (size_t)c * nseg + b0, lens, (size_t)n * 4, cudaMemcpyDeviceToDevice);
        }
        cudaError_t e = cudaMemcpy(tot, d_total, 8, cudaMemcpyDeviceToHost);
        if (e != cudaSuccess) return cuda_fail(e, "synth batch", __FILE__, __LINE__);
        return OG_OK;
    };
    uint64_t est = 0;
    for (uint32_t c = 0; c < ncol1; c++) {
        unsigned long long tot = 0;
        if ((rc = run_batch(c, 0, batch, nullptr, 0, 0, &tot))) return rc;
        avg[c] = (double)tot / batch;
        est += (uint64_t)(avg[c] * 1.02 * nseg) + (1u << 20);
    }
    s->data_len = est;
    if ((rc = dalloc(&s->d_data, est + 1024))) return rc;
    s->owns_data = true;
    uint64_t base = 0;
    for (uint32_t c = 0; c < ncol1; c++) {
        for (uint32_t b0 = 0; b0 < nseg; b0 += batch) {
            uint32_t n = std::min(batch, nseg - b0);
            unsigned long long tot = 0;
            if ((rc = run_batch(c, b0, n, s->d_data, base, est, &tot))) return rc;
            base += tot;
            if (base > est) { set_error("synthetic blob estimate too small"); return OG_E_NOMEM; }
        }
    }
    int fl = 0;
    CU(cudaMemcpy(&fl, flags, 4, cudaMemcpyDeviceToHost));
    if (fl & 16) { set_error("synthetic blob overflow"); return OG_E_NOMEM; }
    CU(cudaMemset(s->d_data + base, 0, std::min<uint64_t>(1024, est + 1024 - base)));
    s->data_len = base;
    if ((rc = shard_finalize(s.get(), false))) return rc;
    *out = s.release();
    return OG_OK;
}

} // extern "C"
