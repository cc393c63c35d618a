/*
 * decode.cuh — device-side page parsing and column block decoders (sm_90a).
 *
 * One thread owns one page and walks it sequentially, handing each decoded value to an `emit(i, bits)` functor,
 * so the same decoders serve the materialise kernels (emit = store) and the fused aggregate kernels
 * (emit = accumulate).  Formats follow SURVEY.md App.A; reference functions replaced:
 *   parse_field_header   engine/immutable/column_builder.go:446-486 DecodeColumnHeader, reader.go:700 DecodeColumnOfOneValue
 *   decode_float_block   lib/compress/float.go:139 AdaptiveDecoding; tsm1/batch_float.go:278 FloatArrayDecodeAll;
 *                        lib/compress/compress.go:51,95 SameValueDecoding / RLE.Decoding
 *   decode_int_block     lib/encoding/int.go:370 Integer.Decoding (:214 const-delta, :256 simple8b, :316 raw)
 *   decode_time_*        lib/encoding/timestamp.go:310 Time.Decoding (:190, :227, :299)
 *   decode_bool_block    lib/encoding/bool.go:63 Boolean.Decoding
 * Unsupported on the device (reported at shard open, never silently skipped): float snappy(2)/mlf(6),
 * int zstd(3), time snappy(3), strings.
 */
#pragma once
#include <cstdint>

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

/* ---------------- MSB-first bit reader over an unaligned byte stream ---------------- */
struct BitReader {
    const uint8_t *p; uint64_t pos; uint64_t nbits;
    __device__ __forceinline__ bool has(unsigned k) const { return pos + k <= nbits; }
    /* next k (1..64) bits, MSB first; caller guarantees has(k) */
    __device__ __forceinline__ uint64_t read(unsigned k) {
        const uint8_t *b = p + (pos >> 3);
        unsigned sh = (unsigned)(pos & 7);
        uint64_t w = ld_be64(b) << sh;
        if (sh && sh + k > 64) w |= (uint64_t)__ldg(b + 8) >> (8 - sh);
        pos += k;
        return w >> (64 - k);
    }
};

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

/* sequential time decode; emit(i, t).  Returns D_OK or D_CORRUPT. */
template <class Emit>
__device__ __forceinline__ int decode_time_values(const TimeDesc &t, Emit &&emit) {
    if (t.kind == 0 || t.kind == 3) {
        uint64_t cur = (uint64_t)t.t0;
        for (uint32_t i = 0; i < t.rows; i++) { emit(i, (int64_t)cur); cur += t.delta; }
        return D_OK;
    }
    if (t.kind == 2) {
        for (uint32_t i = 0; i < t.rows; i++) emit(i, zigzag_dec(ld_be64(t.words + 8ull * i)));
        return D_OK;
    }
    uint64_t cur = (uint64_t)t.t0; uint32_t idx = 0;
    emit(idx++, (int64_t)cur);
    for (uint32_t w = 0; w < t.n_words; w++) {
        uint64_t v = ld_be64(t.words + 8ull * w);
        unsigned n, bits; s8b_sel((unsigned)(v >> 60), n, bits);
        uint64_t mask = bits == 0 ? 0 : ((1ull << bits) - 1);
        for (unsigned k = 0; k < n; k++) {
            if (idx >= t.rows) return D_CORRUPT;
            uint64_t d = bits == 0 ? 1ull : ((v >> (k * bits)) & mask);
            cur += d * t.delta;
            emit(idx++, (int64_t)cur);
        }
    }
    return idx == t.rows ? D_OK : D_CORRUPT;
}

/* ---------------- float blocks ---------------- */
#define OG_UVNAN 0x7FF8000000000001ull

/* n = number of non-null values expected (rows - nilCount).  emit(i, bits). */
template <class Emit>
__device__ __forceinline__ int decode_float_block(const uint8_t *in, uint32_t len, uint32_t n, Emit &&emit) {
    if (n == 0) return D_OK;
    if (len < 1) return D_CORRUPT;
    int algo = __ldg(in) >> 4;
    const uint8_t *b = in + 1; uint32_t bl = len - 1;
    switch (algo) {
    case 0: { /* floatCompressedNull: raw LE */
        if (bl < 8ull * n) return D_CORRUPT;
        for (uint32_t i = 0; i < n; i++) emit(i, ld_le64(b + 8ull * i));
        return D_OK;
    }
    case 3: { /* Gorilla: [0x10][8 B BE first][bit stream] */
        if (bl < 9) return D_CORRUPT;
        uint64_t val = ld_be64(b + 1);
        if (val == OG_UVNAN) return D_CORRUPT; /* empty stream but values expected */
        emit(0, val);
        BitReader br{b + 9, 0, (uint64_t)(bl - 9) * 8};
        unsigned trailing = 0, meaningful = 64;
        for (uint32_t i = 1; i < n; i++) {
            if (!br.has(1)) return D_CORRUPT;
            if (br.read(1)) {
                if (!br.has(1)) return D_CORRUPT;
                if (br.read(1)) {
                    if (!br.has(11)) return D_CORRUPT;
                    unsigned lm = (unsigned)br.read(11);
                    unsigned leading = (lm >> 6) & 0x1f;
                    meaningful = lm & 0x3f;
                    if (meaningful > 0) { if (leading + meaningful > 64) return D_CORRUPT; trailing = 64 - leading - meaningful; }
                    else { trailing = 0; meaningful = 64; }
                }
                if (!br.has(meaningful)) return D_CORRUPT;
                val ^= br.read(meaningful) << trailing;
                if (val == OG_UVNAN) return D_CORRUPT; /* sentinel before n values */
            }
            emit(i, val);
        }
        return D_OK;
    }
    case 4: { /* Same: [u16 BE count][8 B LE value, absent when 0] */
        if (bl < 2) return D_CORRUPT;
        uint32_t cnt = ld_be16(b);
        if (cnt != n) return D_CORRUPT;
        uint64_t v = 0;
        if (bl != 2) { if (bl < 10) return D_CORRUPT; v = ld_le64(b + 2); }
        for (uint32_t i = 0; i < n; i++) emit(i, v);
        return D_OK;
    }
    case 5: { /* RLE: repeat [u16 BE n (bit15 = zero run)][8 B LE] */
        uint32_t idx = 0;
        while (bl >= 2) {
            uint32_t c = ld_be16(b);
            uint64_t v = 0;
            if (c >> 15) { c -= 1u << 15; b += 2; bl -= 2; }
            else { if (bl < 10) return D_CORRUPT; v = ld_le64(b + 2); b += 10; bl -= 10; }
            if (idx + c > n) return D_CORRUPT;
            for (uint32_t k = 0; k < c; k++) emit(idx++, v);
        }
        return idx == n ? D_OK : D_CORRUPT;
    }
    case 1: case 2: case 6: return D_UNSUPPORTED; /* legacy gorilla, snappy, mlf */
    default: return D_CORRUPT;
    }
}

/* ---------------- int blocks ---------------- */
template <class Emit>
__device__ __forceinline__ int decode_int_block(const uint8_t *in, uint32_t len, uint32_t n, Emit &&emit) {
    if (n == 0) return D_OK;
    if (len < 5) return D_CORRUPT;
    int ty = __ldg(in) >> 4;
    const uint8_t *b = in + 1; uint32_t bl = len - 1;
    switch (ty) {
    case 4: { /* raw: [u32 byteLen][n x u64 BE zigzag] */
        uint32_t byte_len = ld_be32(b);
        if (bl - 4 < byte_len || (bl - 4) / 8 != n) return D_CORRUPT;
        for (uint32_t i = 0; i < n; i++) emit(i, (uint64_t)zigzag_dec(ld_be64(b + 4 + 8ull * i)));
        return D_OK;
    }
    case 1: { /* const delta */
        if (bl < 8) return D_CORRUPT;
        uint64_t first = ld_be64(b), d, c;
        int k = ld_uvarint(b + 8, bl - 8, &d);
        if (k == 0) return D_CORRUPT;
        int k2 = ld_uvarint(b + 8 + k, bl - 8 - k, &c);
        if (k2 == 0 || c + 1 != n) return D_CORRUPT;
        uint64_t cur = (uint64_t)zigzag_dec(first), dv = (uint64_t)zigzag_dec(d);
        for (uint32_t i = 0; i < n; i++) { emit(i, cur); cur += dv; }
        return D_OK;
    }
    case 2: { /* simple8b: [u32 encCnt][u32 srcCnt][u64 BE zz(v0)][words] */
        if (bl < 16) return D_CORRUPT;
        uint32_t enc = ld_be32(b), src = ld_be32(b + 4);
        if (src != n || enc == 0 || bl - 8 < enc * 8ull) return D_CORRUPT;
        uint64_t cur = (uint64_t)zigzag_dec(ld_be64(b + 8));
        uint32_t idx = 0;
        emit(idx++, cur);
        const uint8_t *w = b + 16;
        for (uint32_t wi = 0; wi + 1 < enc; wi++) {
            uint64_t v = ld_be64(w + 8ull * wi);
            unsigned cnt, bits; s8b_sel((unsigned)(v >> 60), cnt, bits);
            uint64_t mask = bits == 0 ? 0 : ((1ull << bits) - 1);
            for (unsigned k = 0; k < cnt; k++) {
                if (idx >= n) return D_CORRUPT;
                uint64_t z = bits == 0 ? 1ull : ((v >> (k * bits)) & mask);
                cur += (uint64_t)zigzag_dec(z);
                emit(idx++, cur);
            }
        }
        return idx == n ? D_OK : D_CORRUPT;
    }
    case 3: return D_UNSUPPORTED; /* zstd */
    default: return D_CORRUPT;
    }
}

/* ---------------- bool blocks ---------------- */
template <class Emit>
__device__ __forceinline__ int decode_bool_block(const uint8_t *in, uint32_t len, uint32_t n, Emit &&emit) {
    if (n == 0) return D_OK;
    if (len < 5) return D_CORRUPT;
    if ((__ldg(in) >> 4) != 1) return D_CORRUPT;
    uint32_t cnt = ld_be32(in + 1);
    if (cnt != n || (uint64_t)(len - 5) * 8 < n) return D_CORRUPT;
    const uint8_t *b = in + 5;
    for (uint32_t i = 0; i < n; i++) emit(i, (uint64_t)((__ldg(b + (i >> 3)) >> (7 - (i & 7))) & 1));
    return D_OK;
}

/* typed dispatch: decodes the n non-null values of a page block */
template <class Emit>
__device__ __forceinline__ int decode_block(int type, const PageHdr &h, Emit &&emit) {
    uint32_t n = h.rows - h.nil_count;
    if (h.one_row) {
        if (n == 0) return D_OK;
        if (type == 5) { emit(0u, (uint64_t)__ldg(h.block)); return D_OK; }
        if (h.block_len < 8) return D_CORRUPT;
        emit(0u, ld_le64(h.block)); return D_OK;
    }
    if (type == 3) return decode_float_block(h.block, h.block_len, n, emit);
    if (type == 1) return decode_int_block(h.block, h.block_len, n, emit);
    if (type == 5) return decode_bool_block(h.block, h.block_len, n, emit);
    return D_UNSUPPORTED;
}

} // namespace ogpu
