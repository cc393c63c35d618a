/*
 * decode.cuh — device-side page parsing and the generic page decoders (sm_90a).
 *
 * One thread owns one segment and pulls its rows in order: TimeIter::next() yields the time of the next row, ColIter::next()
 * the (valid, value) of the next row of one field column, straight from the page bytes.  Every generic consumer — shard
 * validation, the materialise kernels, the decode step of the tile path and the pull-iterator aggregate kernel — uses these
 * two iterators, so they all agree on what a corrupt page is.  A consumer that walks a page to its last row calls finish(),
 * which checks that the words / runs hold exactly the page's value count.  k_fused_cols (fused_cols.cuh) decodes Gorilla,
 * Simple8b and bool pages in loops of its own and pulls the other codecs through ColIter::value(); a pass of it that reaches a
 * segment's last row runs the same checks (finish() for the ColIter codecs, their restatement for its Simple8b loop).  Shard
 * open (k_validate) guarantees that a page's validity bits mark exactly
 * rows - nil_count rows valid, so no iterator takes more values from a block than its header counts.  Formats follow
 * SURVEY.md App.A; reference functions replaced:
 *   parse_field_header   engine/immutable/column_builder.go:446-486 DecodeColumnHeader, reader.go:700 DecodeColumnOfOneValue
 *   ColIter (float)      lib/compress/float.go:139 AdaptiveDecoding; tsm1/batch_float.go:278 FloatArrayDecodeAll;
 *                        lib/compress/compress.go:51,95 SameValueDecoding / RLE.Decoding
 *   ColIter (int)        lib/encoding/int.go:370 Integer.Decoding (:214 const-delta, :256 simple8b, :316 raw)
 *   ColIter (bool)       lib/encoding/bool.go:63 Boolean.Decoding
 *   parse_time_page, TimeIter   lib/encoding/timestamp.go:310 Time.Decoding (:190, :227, :299)
 * Unsupported on the device (reported at shard open, never silently skipped): float snappy(2)/mlf(6),
 * int zstd(3), time snappy(3), string values.
 */
#pragma once
#include <cstdint>
#include "../../include/ogpu.h"

namespace ogpu {

enum { D_OK = 0, D_UNSUPPORTED = 1, D_CORRUPT = 2, D_TYPE = 3, D_WATCHDOG = 4, D_SNAPPY = 5 /* internal: Snappy page, transcoded to a raw page when the shard is opened */ /* a device-side progress guard fired (reported as OG_E_CUDA) */ };

/* ---------------- unaligned big-endian loads on top of aligned 64-bit __ldg ---------------- */
__device__ __forceinline__ uint64_t bswap64(uint64_t v) {
    uint32_t lo = (uint32_t)v, hi = (uint32_t)(v >> 32);
    return ((uint64_t)__byte_perm(lo, 0, 0x0123) << 32) | (uint64_t)__byte_perm(hi, 0, 0x0123);
}
/* little-endian 64-bit value of bytes p[0..7]; p may be unaligned. Reads up to 15 bytes past p rounded to words:
 * every page buffer carries >= 16 bytes of tail padding (see api.cu). */
__device__ __forceinline__ uint64_t ld_le64(const uint8_t *p) {
    uintptr_t a = (uintptr_t)p;
    const uint64_t *q = (const uint64_t *)(a & ~(uintptr_t)7);
    unsigned sh = (unsigned)(a & 7) * 8;
    uint64_t lo = __ldg(q);
    if (sh == 0) return lo;
    uint64_t hi = __ldg(q + 1);
    return (lo >> sh) | (hi << (64 - sh));
}
__device__ __forceinline__ uint64_t ld_be64(const uint8_t *p) { return bswap64(ld_le64(p)); }
__device__ __forceinline__ uint32_t ld_be32(const uint8_t *p) {
    return ((uint32_t)__ldg(p) << 24) | ((uint32_t)__ldg(p + 1) << 16) | ((uint32_t)__ldg(p + 2) << 8) | (uint32_t)__ldg(p + 3);
}
__device__ __forceinline__ uint32_t ld_be16(const uint8_t *p) { return ((uint32_t)__ldg(p) << 8) | (uint32_t)__ldg(p + 1); }

/* encoding/binary.Uvarint; returns bytes consumed or 0 on error */
__device__ __forceinline__ int ld_uvarint(const uint8_t *p, uint32_t len, uint64_t *out) {
    uint64_t x = 0; unsigned s = 0;
    for (uint32_t i = 0; i < len && i < 10; i++) {
        uint8_t c = __ldg(p + i);
        if (c < 0x80) { *out = x | ((uint64_t)c << s); return (int)i + 1; }
        x |= (uint64_t)(c & 0x7f) << s; s += 7;
    }
    return 0;
}
__device__ __forceinline__ int64_t zigzag_dec(uint64_t u) { return (int64_t)(u >> 1) ^ -(int64_t)(u & 1); }

/* ---------------- Snappy block format (golang/snappy, klauspost/compress snappy: lib/compress/compress.go:132-144) ----------------
 * [uvarint decoded length] then elements: tag&3 == 0 literal (len-1 in the upper six bits, 60..63 = 1..4 length bytes follow),
 * 1 copy with 11-bit offset (len 4..11), 2 copy with 16-bit offset, 3 copy with 32-bit offset (len 1..64).
 * One thread decodes one block into `out` (load-time transcode of Snappy pages, api.cu); returns D_OK / D_CORRUPT. */
__device__ __forceinline__ int snappy_decoded_len(const uint8_t *in, uint32_t len, uint32_t *n, uint32_t *hdr) {
    uint64_t v; int k = ld_uvarint(in, len, &v);
    if (k <= 0 || v > 0xffffffffull) return D_CORRUPT;
    *n = (uint32_t)v; *hdr = (uint32_t)k;
    return D_OK;
}
__device__ inline int snappy_decode_dev(const uint8_t *in, uint32_t len, uint8_t *out, uint32_t out_cap, uint32_t *out_len) {
    uint32_t dlen, s;
    if (snappy_decoded_len(in, len, &dlen, &s) != D_OK || dlen > out_cap) return D_CORRUPT;
    uint32_t d = 0;
    while (s < len) {
        const uint32_t tag = __ldg(in + s);
        uint32_t length, offset;
        switch (tag & 3) {
        case 0: {
            uint32_t x = tag >> 2;
            if (x < 60) s += 1;
            else {
                const uint32_t nb = x - 59;
                if (s + 1 + nb > len) return D_CORRUPT;
                x = 0;
                for (uint32_t i = 0; i < nb; i++) x |= (uint32_t)__ldg(in + s + 1 + i) << (8 * i);
                s += 1 + nb;
            }
            length = x + 1;
            if (length == 0 || length > len - s || length > dlen - d) return D_CORRUPT;
            for (uint32_t i = 0; i < length; i++) out[d + i] = __ldg(in + s + i);
            d += length; s += length;
            continue;
        }
        case 1:
            if (s + 2 > len) return D_CORRUPT;
            length = 4 + ((tag >> 2) & 7); offset = ((tag & 0xe0) << 3) | __ldg(in + s + 1); s += 2;
            break;
        case 2:
            if (s + 3 > len) return D_CORRUPT;
            length = 1 + (tag >> 2); offset = __ldg(in + s + 1) | ((uint32_t)__ldg(in + s + 2) << 8); s += 3;
            break;
        default:
            if (s + 5 > len) return D_CORRUPT;
            length = 1 + (tag >> 2);
            offset = __ldg(in + s + 1) | ((uint32_t)__ldg(in + s + 2) << 8) | ((uint32_t)__ldg(in + s + 3) << 16) | ((uint32_t)__ldg(in + s + 4) << 24); s += 5;
            break;
        }
        if (offset == 0 || offset > d || length > dlen - d) return D_CORRUPT;
        for (uint32_t i = 0; i < length; i++) out[d + i] = out[d + i - offset]; /* byte by byte: overlapping copies repeat a pattern */
        d += length;
    }
    if (d != dlen) return D_CORRUPT;
    *out_len = d;
    return D_OK;
}

/* ---------------- column segment header ---------------- */
struct PageHdr {
    uint32_t rows;          /* Len */
    uint32_t nil_count;
    const uint8_t *bitmap;  /* validity bits, LSB-first at bit bm_off+i; nullptr = all valid (Full) / all null (Empty) */
    uint32_t bm_off;
    const uint8_t *block;   /* encoded non-null values */
    uint32_t block_len;
    uint8_t one_row;        /* BlockXxxOne: block holds the raw LE value */
};

/* seg_rows = row count of the segment taken from its time page (a normal header does not store Len:
 * reader.go:511 derives rows = len(values) + nilCount; the time page always knows it). */
__device__ __forceinline__ int parse_field_header(const uint8_t *p, uint32_t len, int col_type, uint32_t seg_rows, PageHdr &h) {
    if (len < 1) return D_CORRUPT;
    uint8_t typ = __ldg(p);
    h.one_row = 0; h.bitmap = nullptr; h.bm_off = 0;
    if (typ > 16 && typ < 21) { /* IsBlockOne */
        h.rows = 1; h.one_row = 1; h.block = p + 1; h.block_len = len - 1;
        h.nil_count = (len == 1) ? 1u : 0u;
        return D_OK;
    }
    if (typ > 30 && typ < 35) { /* IsBlockFull */
        if (len < 5) return D_CORRUPT;
        h.rows = ld_be32(p + 1); h.nil_count = 0; h.block = p + 5; h.block_len = len - 5;
        return D_OK;
    }
    if (typ > 40 && typ < 45) { /* IsBlockEmpty */
        if (len < 5) return D_CORRUPT;
        h.rows = ld_be32(p + 1); h.nil_count = h.rows; h.block = p + 5; h.block_len = 0;
        return D_OK;
    }
    if (typ != (uint8_t)col_type) return D_TYPE;
    if (len < 13) return D_CORRUPT;
    uint32_t nb = ld_be32(p + 1);
    if (13ull + (uint64_t)nb > (uint64_t)len) return D_CORRUPT; /* 64-bit: nb near 2^32 must not wrap the bound */
    h.bitmap = p + 5;
    h.bm_off = ld_be32(p + 5 + nb);
    h.nil_count = ld_be32(p + 9 + nb);
    h.block = p + 13 + nb; h.block_len = len - 13 - nb;
    h.rows = seg_rows;
    /* the validity bits of the rows must lie inside the bitmap, and a page cannot hold more nulls than rows */
    if (h.nil_count > seg_rows || ((uint64_t)h.bm_off + seg_rows + 7) / 8 > (uint64_t)nb) return D_CORRUPT;
    return D_OK;
}
__device__ __forceinline__ bool hdr_row_valid(const PageHdr &h, uint32_t i) {
    if (!h.bitmap) return h.nil_count == 0;
    uint32_t b = h.bm_off + i;
    return (__ldg(h.bitmap + (b >> 3)) >> (b & 7)) & 1;
}
/* number of rows the validity bits mark valid (a page with a bitmap) */
__device__ __forceinline__ uint32_t hdr_valid_rows(const PageHdr &h) {
    uint32_t n = 0;
    for (uint32_t i = 0; i < h.rows;) {
        const uint32_t b = h.bm_off + i, k = min(8u - (b & 7), h.rows - i);
        n += __popc((__ldg(h.bitmap + (b >> 3)) >> (b & 7)) & ((1u << k) - 1));
        i += k;
    }
    return n;
}

/* ---------------- time pages ---------------- */
struct TimeDesc {
    int kind;        /* 0 const-delta (closed form), 1 simple8b, 2 raw zigzag BE, 3 one-row */
    uint32_t rows;
    int64_t t0;
    uint64_t delta;  /* const-delta step, or simple8b scale */
    const uint8_t *words; uint32_t n_words; /* simple8b words after t0 / raw values */
};
__device__ __forceinline__ int parse_time_page(const uint8_t *p, uint32_t len, TimeDesc &t) {
    if (len < 1) return D_CORRUPT;
    uint8_t typ = __ldg(p);
    if (typ == 18) { /* BlockIntegerOne: raw LE int64 */
        if (len < 9) return D_CORRUPT;
        t.kind = 3; t.rows = 1; t.t0 = (int64_t)ld_le64(p + 1); t.delta = 0; return D_OK;
    }
    if (typ != 32 || len < 10) return (typ == 1 || typ == 42) ? D_UNSUPPORTED : D_CORRUPT; /* time columns are always Full */
    t.rows = ld_be32(p + 1);
    const uint8_t *b = p + 5; uint32_t bl = len - 5;
    int tag = __ldg(b) >> 4;
    b++; bl--;
    if (tag == 1) { /* constDeltaDecoding :190 */
        if (bl < 8) return D_CORRUPT;
        t.kind = 0; t.t0 = (int64_t)ld_be64(b);
        uint64_t d, c; int k = ld_uvarint(b + 8, bl - 8, &d);
        if (k == 0) return D_CORRUPT;
        int k2 = ld_uvarint(b + 8 + k, bl - 8 - k, &c);
        if (k2 == 0) return D_CORRUPT;
        t.delta = d;
        if (c + 1 != t.rows) return D_CORRUPT;
        return D_OK;
    }
    if (tag == 2) { /* simple8bDecoding :227 */
        if (bl < 24) return D_CORRUPT;
        t.kind = 1; t.delta = ld_be64(b);
        uint32_t enc = ld_be32(b + 8), src = ld_be32(b + 12);
        if (src != t.rows || bl - 16 < enc * 8ull || enc == 0) return D_CORRUPT;
        t.t0 = (int64_t)ld_be64(b + 16); t.words = b + 24; t.n_words = enc - 1;
        return D_OK;
    }
    if (tag == 4) { /* unpackUncompressedData :299 */
        if (bl < 4) return D_CORRUPT;
        uint32_t byte_len = ld_be32(b);
        if (bl - 4 < byte_len) return D_CORRUPT;
        t.kind = 2; t.words = b + 4; t.n_words = (bl - 4) / 8;
        if (t.n_words != t.rows) return D_CORRUPT;
        t.t0 = t.n_words ? zigzag_dec(ld_be64(t.words)) : 0; t.delta = 0;
        return D_OK;
    }
    return tag == 3 ? D_SNAPPY : D_CORRUPT; /* snappyDecoding :274: transcoded at shard open */
}

/* simple8b selector table (simple8b/encoding.go:193-210) */
__device__ __forceinline__ void s8b_sel(unsigned sel, unsigned &n, unsigned &bits) {
    const unsigned N[16] = {240, 120, 60, 30, 20, 15, 12, 10, 8, 7, 6, 5, 4, 3, 2, 1};
    const unsigned B[16] = {0, 0, 1, 2, 3, 4, 5, 6, 7, 8, 10, 12, 15, 20, 30, 60};
    n = N[sel]; bits = B[sel];
}

/* time of the next row of a time page; rows past t.rows must not be pulled */
struct TimeIter {
    TimeDesc d; uint64_t cur; uint32_t idx; uint32_t w; unsigned k, n, bits; uint64_t word;
    int err;
    __device__ __forceinline__ void init(const TimeDesc &t) { d = t; cur = (uint64_t)t.t0; idx = 0; w = 0; k = 0; n = 0; bits = 0; word = 0; err = D_OK; }
    __device__ __forceinline__ int64_t next() { /* time of row idx, then advance */
        int64_t t;
        if (d.kind == 0 || d.kind == 3) { t = (int64_t)cur; cur += d.delta; }
        else if (d.kind == 2) { t = zigzag_dec(ld_be64(d.words + 8ull * idx)); }
        else {
            if (idx != 0) {
                while (k == n) { /* next simple8b word */
                    if (w >= d.n_words) { err = D_CORRUPT; idx++; return (int64_t)cur; } /* fewer deltas than rows */
                    word = ld_be64(d.words + 8ull * w); w++;
                    s8b_sel((unsigned)(word >> 60), n, bits); k = 0;
                }
                uint64_t dv = bits == 0 ? 1ull : ((word >> (k * bits)) & ((1ull << bits) - 1));
                k++;
                cur += dv * d.delta;
            }
            t = (int64_t)cur;
        }
        idx++;
        return t;
    }
    /* after the last row: a Simple8b page holds exactly rows - 1 deltas (timestamp.go:267) */
    __device__ __forceinline__ void finish() {
        if (d.kind == 1 && (w != d.n_words || k != n)) err = D_CORRUPT;
    }
};

/* ---------------- field pages ---------------- */
#define OG_UVNAN 0x7FF8000000000001ull

/* next (valid, value) of one field column of one segment; value = raw 64-bit cell (double bits / int64 / bool 0,1) */
struct ColIter {
    enum { K_ABSENT = 0, K_NULLMAP /* string column: validity only, values are never decoded */, K_ONE, K_F_RAW, K_F_GORILLA, K_F_SAME, K_F_RLE, K_I_CONST, K_I_S8B, K_I_RAW, K_B_BITS };
    PageHdr h;
    int kind, type;
    uint32_t row;      /* next row */
    uint32_t idx;      /* next non-null value */
    const uint8_t *p;  /* payload cursor (codec specific) */
    uint64_t cur;      /* current value / run value / accumulator */
    uint64_t aux;      /* gorilla: bit position; s8b: current word; const: delta */
    uint32_t a, b, c;  /* gorilla: trailing, meaningful, bits in stream; s8b: k, n, bits; rle: run left, -, bytes left */
    uint32_t words_left;
    int err;

    __device__ __forceinline__ void init(const uint8_t *page, uint32_t len, int col_type, uint32_t seg_rows) {
        type = col_type; row = 0; idx = 0; err = D_OK; cur = 0; aux = 0; a = b = c = 0; words_left = 0; p = nullptr;
        if (len == 0) { kind = K_ABSENT; h.rows = seg_rows; h.nil_count = seg_rows; h.bitmap = nullptr; h.bm_off = 0; h.block = nullptr; h.block_len = 0; h.one_row = 0; return; }
        int rc = parse_field_header(page, len, col_type, seg_rows, h);
        if (rc != D_OK) { err = rc; kind = K_ABSENT; return; }
        const uint32_t n = h.rows - h.nil_count;
        if (n == 0) { kind = K_ABSENT; return; }
        if (col_type == OG_TYPE_STRING) { kind = K_NULLMAP; return; } /* lib/encoding/string.go:286-302 is not needed for count(): ValidCount reads the bitmap */
        if (h.one_row) { kind = K_ONE; cur = col_type == OG_TYPE_BOOL ? (uint64_t)__ldg(h.block) : (h.block_len >= 8 ? ld_le64(h.block) : 0); if (col_type != OG_TYPE_BOOL && h.block_len < 8) err = D_CORRUPT; return; }
        if (h.block_len < 1) { err = D_CORRUPT; kind = K_ABSENT; return; }
        const uint8_t *in = h.block; const uint32_t bl = h.block_len - 1;
        const int tag = __ldg(in) >> 4;
        p = in + 1;
        if (col_type == OG_TYPE_FLOAT) {
            switch (tag) {
            case 0: kind = K_F_RAW; if (bl < 8ull * n) err = D_CORRUPT; break;
            case 3: kind = K_F_GORILLA;
                if (bl < 9) { err = D_CORRUPT; break; }
                cur = ld_be64(p + 1); p += 9; aux = 0; a = 0; b = 64; c = (bl - 9) * 8;
                if (cur == OG_UVNAN) err = D_CORRUPT;
                break;
            case 4: kind = K_F_SAME; if (bl < 2 || ld_be16(p) != n) { err = D_CORRUPT; break; } cur = 0; if (bl != 2) { if (bl < 10) err = D_CORRUPT; else cur = ld_le64(p + 2); } break;
            case 5: kind = K_F_RLE; a = 0; c = bl; break;
            default: err = (tag == 1 || tag == 2 || tag == 6) ? D_UNSUPPORTED : D_CORRUPT; break;
            }
        } else if (col_type == OG_TYPE_INT) {
            if (bl < 4) { err = D_CORRUPT; kind = K_ABSENT; return; }
            switch (tag) {
            case 4: kind = K_I_RAW; if (bl - 4 < ld_be32(p) || (bl - 4) / 8 != n) err = D_CORRUPT; p += 4; break;
            case 1: { kind = K_I_CONST;
                if (bl < 8) { err = D_CORRUPT; break; }
                uint64_t d, cnt; int k = ld_uvarint(p + 8, bl - 8, &d);
                int k2 = k ? ld_uvarint(p + 8 + k, bl - 8 - k, &cnt) : 0;
                if (k == 0 || k2 == 0 || cnt + 1 != n) { err = D_CORRUPT; break; }
                cur = (uint64_t)zigzag_dec(ld_be64(p)); aux = (uint64_t)zigzag_dec(d);
                break; }
            case 2: { kind = K_I_S8B;
                if (bl < 16) { err = D_CORRUPT; break; }
                const uint32_t enc = ld_be32(p), src = ld_be32(p + 4);
                if (src != n || enc == 0 || bl - 8 < enc * 8ull) { err = D_CORRUPT; break; }
                cur = (uint64_t)zigzag_dec(ld_be64(p + 8)); p += 16; words_left = enc - 1; a = 0; b = 0; c = 0;
                break; }
            default: err = tag == 3 ? D_UNSUPPORTED : D_CORRUPT; break;
            }
        } else if (col_type == OG_TYPE_BOOL) {
            kind = K_B_BITS;
            if (tag != 1 || bl < 4 || ld_be32(p) != n || (uint64_t)(bl - 4) * 8 < n) err = D_CORRUPT;
            p += 4;
        } else err = D_UNSUPPORTED;
        if (err != D_OK) kind = K_ABSENT;
    }

    /* value of the next non-null row (idx-th value of the block) */
    __device__ __forceinline__ uint64_t value() {
        const uint32_t i = idx++;
        switch (kind) {
        case K_ONE: return cur;
        case K_F_RAW: return ld_le64(p + 8ull * i);
        case K_F_SAME: return cur;
        case K_F_GORILLA: {
            if (i == 0) return cur;
            /* one record of tsm1.FloatArrayDecodeAll (batch_float.go:352-508).  '0' (same value) and '10' (window reuse) are
             * handled without a branch — a '0' is a record with zero meaningful bits — so lanes of a warp that sit on different
             * record kinds do not serialise; only the rare '11' (new window) branches. */
            const uint8_t *bp = p + (aux >> 3);
            const unsigned sh = (unsigned)(aux & 7);
            const uint64_t w = ld_be64(bp) << sh; /* >= 57 valid bits */
            unsigned used = (w >> 63) ? 2u : 1u;
            if ((w >> 62) == 3) {
                const unsigned lm = (unsigned)(w >> 51) & 0x7ff;
                const unsigned lead = (lm >> 6) & 0x1f;
                b = lm & 0x3f;
                if (b > 0) { if (lead + b > 64) { err = D_CORRUPT; b = 64; a = 0; } else a = 64 - lead - b; }
                else { a = 0; b = 64; }
                used = 13;
            }
            const unsigned mb = (w >> 63) ? b : 0u; /* meaningful bits of this record */
            aux += used;
            const uint8_t *q2 = p + (aux >> 3);
            const unsigned s2 = (unsigned)(aux & 7);
            uint64_t v = ld_be64(q2) << s2;
            if (s2 + mb > 64) v |= (uint64_t)__ldg(q2 + 8) >> (8 - s2);
            v = mb == 64 ? v : mb == 0 ? 0ull : (v >> (64 - mb));
            aux += mb;
            if (aux > c) { err = D_CORRUPT; aux = c; return cur; } /* truncated stream: later rows keep reading at its end, not past it */
            cur ^= v << a;
            if (mb && cur == OG_UVNAN) err = D_CORRUPT; /* sentinel before the block's value count */
            return cur; }
        case K_F_RLE: {
            while (a == 0) { /* next run: [u16 BE n (bit15 = zero run)][8 B LE] (compress.go:95-120) */
                if (c < 2) { err = D_CORRUPT; return 0; }
                const uint32_t n = ld_be16(p);
                if (n >> 15) { a = n - (1u << 15); cur = 0; p += 2; c -= 2; } /* a zero run of length 0 pads nothing (:105-110) */
                else { /* a value run of length 0 has no defined result in paddingBuffer (:171-187) */
                    if (c < 10 || n == 0) { err = D_CORRUPT; return 0; }
                    a = n; cur = ld_le64(p + 2); p += 10; c -= 10;
                }
            }
            a--;
            return cur; }
        case K_I_RAW: return (uint64_t)zigzag_dec(ld_be64(p + 8ull * i));
        case K_I_CONST: { const uint64_t v = cur; cur += aux; return v; }
        case K_I_S8B: {
            if (i == 0) return cur;
            while (a == b) { /* next simple8b word (simple8b/encoding.go:193-210) */
                if (words_left == 0) { err = D_CORRUPT; return cur; }
                aux = ld_be64(p); p += 8; words_left--;
                unsigned nn, bits; s8b_sel((unsigned)(aux >> 60), nn, bits);
                b = nn; c = bits; a = 0;
            }
            const uint64_t z = c == 0 ? 1ull : ((aux >> (a * c)) & ((1ull << c) - 1));
            a++;
            cur += (uint64_t)zigzag_dec(z);
            return cur; }
        case K_B_BITS: return (uint64_t)((__ldg(p + (i >> 3)) >> (7 - (i & 7))) & 1);
        default: return 0;
        }
    }
    __device__ __forceinline__ bool next(uint64_t &v) {
        const uint32_t r = row++;
        if (kind == K_ABSENT) return false;
        if (!hdr_row_valid(h, r)) return false;
        v = value();
        return true;
    }
    /* after the last row: the words / runs must hold exactly the block's value count */
    __device__ __forceinline__ void finish() {
        const uint32_t n = h.rows - h.nil_count;
        if (kind == K_I_S8B) { /* every slot of every word taken, and as many values as srcCount (int.go:296) */
            if (idx != n || a != b || words_left != 0) err = D_CORRUPT;
        } else if (kind == K_F_RLE) { /* runs add up to n; only zero-length zero runs may follow, and < 2 bytes (compress.go:99-101) */
            if (idx != n || a != 0) err = D_CORRUPT;
            for (; c >= 2 && err == D_OK; p += 2, c -= 2) if (ld_be16(p) != 0x8000u) err = D_CORRUPT;
        }
    }
};

} // namespace ogpu
