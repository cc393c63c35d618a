/*
 * tssp.cpp — the TSSP container.  Read side: file bytes -> og_shard_desc (the flattened ChunkMeta directory og_shard_open
 * takes).  Write side (tssp_build_tail, at the end of the file): everything of a file that follows its chunks, for
 * og_shard_write_tssp (tssp_write.cu lays out and checksums the chunks on the device).  Host code only: the container is a few
 * bytes of metadata per segment, walked once per file; the pages it points at are what the GPU reads and writes.
 *
 * What the reference does on this path (engine/immutable):
 *   file     = "53ac2021" | u64 BE version=2 | chunks | chunk-meta blocks | meta index | bloom | id-time | trailer | footer
 *              (msbuilder.go:1355-1425 Flush, table.go:24-28)
 *   footer   = i64 (zig-zag, BE) trailer offset                                  (msbuilder.go:1413-1415)
 *   trailer  = 6 x i64zz {dataOffset,dataSize,indexSize,metaIndexSize,bloomSize,idTimeSize} + TableStat
 *              (trailer.go:59-88, table_stat.go:36-84) with the ExtraData flags (table_stat.go:122-207)
 *   meta idx = metaIndexItemNum x {u64 id, i64zz minT, i64zz maxT, i64zz offset, u32 count, u32 size}  (tssp_file_meta.go:769-802)
 *   block    = count ChunkMetas back to back, then count x u32 BE start offsets   (msbuilder.go:1481-1500, tssp_file.go:606-658)
 *   chunk    = u64 sid, i64zz offset, u32 size, u32 columnCount, u32 segCount, segCount x (i64zz min, i64zz max),
 *              then per column u16 nameLen, name, u8 type, u16 preAggLen, preAgg, segCount x (i64zz offset, u32 size)
 *              (tssp_file_meta.go:566-581, 228-246, 86-104, 129-143); columns sorted by name, time last
 *   a chunk's bytes = per column [u32 crc][pages of its segments]; Segment.offset is the absolute file offset of a page
 *              (chunkdata_builder_ts.go:37-82)
 * Integers of type int64 are zig-zag coded before the big-endian store (lib/numberenc/number.go:155-168).
 *
 * Not handled (refused with OG_E_UNSUPPORTED): compressed chunk metas (ChunkMetaCompressFlag != 0, chunk_meta_codec.go), detached
 * (object-store) files.  The per-column CRC32 is not verified: pages are validated structurally on the device at og_shard_open.
 */
#include <algorithm>
#include <cmath>
#include <cstring>
#include <map>
#include <memory>
#include <string>
#include <vector>

#include "../../include/ogpu.h"
#include "tssp_write.h"

namespace ogpu { void set_error(const char *fmt, ...); }
using ogpu::set_error;

namespace {

struct Rd { /* bounds-checked big-endian reader over [p, end) */
    const uint8_t *p, *end; bool ok = true;
    Rd(const uint8_t *b, uint64_t n) : p(b), end(b + n) {}
    uint64_t left() const { return (uint64_t)(end - p); }
    bool need(uint64_t n) { if (!ok || left() < n) { ok = false; return false; } return true; }
    uint64_t u64() { if (!need(8)) return 0; uint64_t v = 0; for (int i = 0; i < 8; i++) v = (v << 8) | p[i]; p += 8; return v; }
    int64_t i64() { const uint64_t u = u64(); return (int64_t)(u >> 1) ^ -(int64_t)(u & 1); }
    uint32_t u32() { if (!need(4)) return 0; uint32_t v = ((uint32_t)p[0] << 24) | ((uint32_t)p[1] << 16) | ((uint32_t)p[2] << 8) | p[3]; p += 4; return v; }
    uint32_t u16() { if (!need(2)) return 0; uint32_t v = ((uint32_t)p[0] << 8) | p[1]; p += 2; return v; }
    uint32_t u8() { if (!need(1)) return 0; return *p++; }
    const uint8_t *bytes(uint64_t n) { if (!need(n)) return nullptr; const uint8_t *r = p; p += n; return r; }
};

struct Col {
    std::string name; int type;
    std::vector<uint64_t> off; std::vector<uint32_t> len;
};

} // namespace

struct og_tssp {
    const uint8_t *file; uint64_t len;
    std::string measurement;
    int64_t min_time = 0, max_time = 0, id_count = 0; uint64_t min_id = 0, max_id = 0;
    std::vector<uint64_t> sids; std::vector<uint32_t> seg_begin;
    std::vector<int64_t> tmin, tmax;
    std::vector<uint64_t> time_off; std::vector<uint32_t> time_len;
    std::vector<Col> cols;
    std::vector<og_column_desc> col_desc;
};

extern "C" {

OG_API int og_tssp_parse(const uint8_t *file, uint64_t len, og_tssp **out) {
    if (!file || !out) { set_error("null argument"); return OG_E_INVAL; }
    *out = nullptr;
    static const char magic[] = "53ac2021";
    const uint64_t header = 16, footer = 8;
    if (len < header + footer || memcmp(file, magic, 8) != 0) { set_error("not a TSSP file (magic)"); return OG_E_CORRUPT; }
    { Rd r(file + 8, 8); const uint64_t v = r.u64(); if (v != 2) { set_error("TSSP version %llu (this reader knows 2)", (unsigned long long)v); return OG_E_UNSUPPORTED; } }
    int64_t toff; { Rd r(file + len - footer, footer); toff = r.i64(); }
    if (toff < (int64_t)header || (uint64_t)toff > len - footer) { set_error("trailer offset %lld outside the file", (long long)toff); return OG_E_CORRUPT; }

    /* ---- trailer ---- */
    Rd t(file + toff, len - footer - (uint64_t)toff);
    const int64_t data_off = t.i64(), data_size = t.i64(), index_size = t.i64(), mi_size = t.i64(), bloom_size = t.i64(), idtime_size = t.i64();
    std::unique_ptr<og_tssp> f(new og_tssp());
    f->file = file; f->len = len;
    f->id_count = t.i64(); f->min_id = t.u64(); f->max_id = t.u64(); f->min_time = t.i64(); f->max_time = t.i64();
    const int64_t mi_items = t.i64();
    (void)t.u64(); (void)t.u64(); /* bloomM, bloomK */
    uint32_t dlen = t.u16();
    if (!t.ok) { set_error("trailer truncated"); return OG_E_CORRUPT; }
    { /* ExtraData: 1 B / 2 B legacy forms, else 8 B LE flags with the real length in the upper 32 bits (table_stat.go:177-207) */
        if (t.left() < dlen) { set_error("trailer extra data truncated"); return OG_E_CORRUPT; }
        uint32_t compress = 0; uint64_t real = dlen;
        if (dlen == 2) compress = t.p[1];
        else if (dlen >= 8) {
            uint64_t fl = 0; for (int i = 7; i >= 0; i--) fl = (fl << 8) | t.p[i];
            compress = (uint32_t)(fl >> 8) & 0xff;
            if ((fl >> 32) != 0) real = fl >> 32;
        }
        if (compress != 0) { set_error("chunk metas are compressed (mode %u): not supported by this reader", compress); return OG_E_UNSUPPORTED; }
        if (!t.bytes(real)) { set_error("trailer extra data truncated"); return OG_E_CORRUPT; }
    }
    { const uint32_t nl = t.u16(); const uint8_t *nm = t.bytes(nl); if (!nm) { set_error("trailer name truncated"); return OG_E_CORRUPT; } f->measurement.assign((const char *)nm, nl); }
    if (data_off != (int64_t)header || data_size < 0 || index_size < 0 || mi_size < 0 || bloom_size < 0 || idtime_size < 0 || mi_items < 0 ||
        (uint64_t)data_off + (uint64_t)data_size + (uint64_t)index_size + (uint64_t)mi_size + (uint64_t)bloom_size + (uint64_t)idtime_size != (uint64_t)toff) {
        set_error("trailer section sizes do not add up to the trailer offset"); return OG_E_CORRUPT;
    }
    const uint64_t index_off = (uint64_t)data_off + (uint64_t)data_size, mi_off = index_off + (uint64_t)index_size;
    if ((uint64_t)mi_items * 40 != (uint64_t)mi_size) { set_error("meta index: %lld items do not fill %lld bytes", (long long)mi_items, (long long)mi_size); return OG_E_CORRUPT; }

    /* ---- meta index -> chunk-meta blocks -> chunk metas ---- */
    std::map<std::string, size_t> col_of;
    Rd mi(file + mi_off, (uint64_t)mi_size);
    uint64_t prev_sid = 0;
    for (int64_t b = 0; b < mi_items; b++) {
        (void)mi.u64(); (void)mi.i64(); (void)mi.i64();
        const int64_t boff = mi.i64(); const uint32_t count = mi.u32(), bsize = mi.u32();
        if (boff < (int64_t)index_off || (uint64_t)boff + bsize > mi_off || (uint64_t)count * 4 >= bsize) { set_error("meta index item %lld points outside the chunk-meta region", (long long)b); return OG_E_CORRUPT; }
        Rd cm(file + boff, bsize - (uint64_t)count * 4);
        for (uint32_t i = 0; i < count; i++) {
            const uint64_t sid = cm.u64();
            (void)cm.i64(); (void)cm.u32();
            const uint32_t ncol = cm.u32(), nseg = cm.u32();
            if (!cm.ok || ncol == 0 || (uint64_t)nseg * 16 > cm.left()) { set_error("chunk meta %u of block %lld is truncated", i, (long long)b); return OG_E_CORRUPT; }
            if (sid == 0 || (!f->sids.empty() && sid <= prev_sid)) { set_error("chunk metas are not in ascending series-id order (sid %llu)", (unsigned long long)sid); return OG_E_CORRUPT; }
            prev_sid = sid;
            const size_t seg0 = f->tmin.size();
            if (seg0 + nseg > 0xffffffffull) { set_error("more than 2^32 segments"); return OG_E_UNSUPPORTED; }
            f->sids.push_back(sid); f->seg_begin.push_back((uint32_t)seg0);
            for (uint32_t s = 0; s < nseg; s++) { f->tmin.push_back(cm.i64()); f->tmax.push_back(cm.i64()); }
            f->time_off.resize(seg0 + nseg, 0); f->time_len.resize(seg0 + nseg, 0);
            for (Col &c : f->cols) { c.off.resize(seg0 + nseg, 0); c.len.resize(seg0 + nseg, 0); }
            for (uint32_t c = 0; c < ncol; c++) {
                const uint32_t nl = cm.u16(); const uint8_t *nm = cm.bytes(nl);
                const int ty = (int)cm.u8(); const uint32_t pl = cm.u16();
                if (!cm.bytes(pl) || (uint64_t)nseg * 12 > cm.left()) { set_error("column meta %u of series %llu is truncated", c, (unsigned long long)sid); return OG_E_CORRUPT; }
                const std::string name((const char *)nm, nl);
                const bool is_time = c + 1 == ncol;
                if (is_time != (name == "time") || (is_time && ty != OG_TYPE_INT)) { set_error("series %llu: the time column must be the last column", (unsigned long long)sid); return OG_E_CORRUPT; }
                uint64_t *off; uint32_t *ln;
                if (is_time) { off = f->time_off.data() + seg0; ln = f->time_len.data() + seg0; }
                else {
                    auto it = col_of.find(name);
                    if (it == col_of.end()) {
                        it = col_of.emplace(name, f->cols.size()).first;
                        Col nc; nc.name = name; nc.type = ty; nc.off.assign(seg0 + nseg, 0); nc.len.assign(seg0 + nseg, 0);
                        f->cols.push_back(std::move(nc));
                    }
                    Col &col = f->cols[it->second];
                    if (col.type != ty) { set_error("column %s changes type inside the file (%d, %d)", name.c_str(), col.type, ty); return OG_E_TYPE; }
                    off = col.off.data() + seg0; ln = col.len.data() + seg0;
                }
                for (uint32_t s = 0; s < nseg; s++) {
                    const int64_t o = cm.i64(); const uint32_t z = cm.u32();
                    if (o < data_off || (uint64_t)o + z > index_off || z == 0) { set_error("series %llu column %s segment %u lies outside the data region", (unsigned long long)sid, name.c_str(), s); return OG_E_CORRUPT; }
                    off[s] = (uint64_t)o; ln[s] = z;
                }
            }
            if (!cm.ok) { set_error("chunk meta of series %llu is truncated", (unsigned long long)sid); return OG_E_CORRUPT; }
        }
        if (cm.left() != 0) { set_error("chunk-meta block %lld: %llu stray bytes", (long long)b, (unsigned long long)cm.left()); return OG_E_CORRUPT; }
    }
    if (!mi.ok) { set_error("meta index truncated"); return OG_E_CORRUPT; }
    f->seg_begin.push_back((uint32_t)f->tmin.size());
    /* schema order: sorted by name (lib/record/record.go:115-123) */
    std::sort(f->cols.begin(), f->cols.end(), [](const Col &a, const Col &b) { return a.name < b.name; });
    for (const Col &c : f->cols) {
        if (c.type != OG_TYPE_INT && c.type != OG_TYPE_FLOAT && c.type != OG_TYPE_BOOL && c.type != OG_TYPE_STRING) { set_error("column %s has type %d", c.name.c_str(), c.type); return OG_E_UNSUPPORTED; }
        og_column_desc d; d.name = c.name.c_str(); d.type = c.type; d.page_off = c.off.data(); d.page_len = c.len.data();
        f->col_desc.push_back(d);
    }
    *out = f.release();
    return OG_OK;
}

OG_API int og_tssp_desc(const og_tssp *f, og_shard_desc *d) {
    if (!f || !d) { set_error("null argument"); return OG_E_INVAL; }
    memset(d, 0, sizeof *d);
    d->data = f->file; d->data_len = f->len;
    d->n_series = (uint32_t)f->sids.size(); d->sids = f->sids.data(); d->series_seg_begin = f->seg_begin.data();
    d->n_segments = (uint32_t)f->tmin.size(); d->seg_tmin = f->tmin.data(); d->seg_tmax = f->tmax.data();
    d->n_columns = (uint32_t)f->col_desc.size(); d->columns = f->col_desc.data();
    d->time_page_off = f->time_off.data(); d->time_page_len = f->time_len.data();
    d->flags = 0;
    return OG_OK;
}

OG_API const char *og_tssp_measurement(const og_tssp *f) { return f ? f->measurement.c_str() : ""; }

OG_API int og_tssp_time_range(const og_tssp *f, int64_t *min_time, int64_t *max_time) {
    if (!f || !min_time || !max_time) { set_error("null argument"); return OG_E_INVAL; }
    *min_time = f->min_time; *max_time = f->max_time;
    return OG_OK;
}

OG_API void og_tssp_free(og_tssp *f) { delete f; }

} // extern "C"

/* =============================================== write side ===============================================
 * What MsBuilder writes behind the chunks (engine/immutable):
 *   ChunkMeta.marshal / ColumnMeta.marshal     tssp_file_meta.go:566-581,228-246; pre-agg blobs pre_aggregation.go marshal()
 *   chunk-meta blocks                          a block closes after 512 metas or once it holds >= 256 KiB (msbuilder.go:348-364,
 *                                              lib/util/util.go:75-76), followed by the u32 start offsets of its metas (:1481-1500)
 *   MetaIndex                                  first sid, time range, offset, count, size of each block (tssp_file_meta.go:769-778)
 *   bloom filter                               msbuilder.go:1336-1353 genBloomFilter over lib/util/lifted/influxdb/pkg/bloom
 *   id-time section                            sequencer.go:332-390 IdTimePairs.Marshal(encTimes = true)
 *   trailer, footer                            trailer.go:58-66, table_stat.go:35-51,125-148, msbuilder.go:1409-1425
 */
namespace {

struct Wr { /* big-endian appender */
    std::vector<uint8_t> &b;
    void u8(uint32_t v) { b.push_back((uint8_t)v); }
    void u16(uint32_t v) { b.push_back((uint8_t)(v >> 8)); b.push_back((uint8_t)v); }
    void u32(uint32_t v) { for (int i = 3; i >= 0; i--) b.push_back((uint8_t)(v >> (8 * i))); }
    void u64(uint64_t v) { for (int i = 7; i >= 0; i--) b.push_back((uint8_t)(v >> (8 * i))); }
    void i64(int64_t v) { u64(((uint64_t)v << 1) ^ (uint64_t)(v >> 63)); } /* zig-zag, lib/numberenc/number.go:156-160 */
    void bytes(const void *p, size_t n) { const uint8_t *q = (const uint8_t *)p; b.insert(b.end(), q, q + n); }
};

/* IntegerPreAgg / FloatPreAgg / BooleanPreAgg / StringPreAgg / TimePreAgg .marshal() with ChunkMetaCompressNone */
void put_preagg(Wr &w, int type, bool is_time, const ogpu::PreAggCell &c) {
    if (is_time) { w.u16(4); w.u32((uint32_t)c.count); return; }
    switch (type) {
    case OG_TYPE_STRING: w.u16(8); w.i64(c.count); return;
    case OG_TYPE_BOOL: w.u16(26); w.i64(c.count); w.i64(c.mint); w.i64(c.maxt); w.u8((uint32_t)c.minv); w.u8((uint32_t)c.maxv); return;
    case OG_TYPE_FLOAT:
        if (c.count == 1) { w.u16(16); w.u64(c.minv); w.i64(c.mint); return; }
        w.u16(48); w.u64(c.minv); w.u64(c.maxv); w.i64(c.mint); w.i64(c.maxt); w.u64(c.sum); w.i64(c.count); return;
    default: /* OG_TYPE_INT */
        if (c.count == 1) { w.u16(16); w.i64((int64_t)c.minv); w.i64(c.mint); return; }
        w.u16(48); w.i64((int64_t)c.minv); w.i64((int64_t)c.maxv); w.i64(c.mint); w.i64(c.maxt); w.i64((int64_t)c.sum); w.i64(c.count); return;
    }
}

/* xxHash64, seed 0, of eight bytes (github.com/cespare/xxhash/v2 Sum64, the hash of the reference's bloom filter) */
uint64_t xxh64_8(const uint8_t *p) {
    const uint64_t P1 = 11400714785074694791ull, P2 = 14029467366897019727ull, P3 = 1609587929392839161ull, P4 = 9650029242287828579ull, P5 = 2870177450012600261ull;
    auto rotl = [](uint64_t x, int r) { return (x << r) | (x >> (64 - r)); };
    uint64_t k = 0; for (int i = 7; i >= 0; i--) k = (k << 8) | p[i];
    uint64_t h = P5 + 8;
    h ^= rotl(k * P2, 31) * P1;
    h = rotl(h, 27) * P1 + P4;
    h ^= h >> 33; h *= P2; h ^= h >> 29; h *= P3; h ^= h >> 32;
    return h;
}

/* genBloomFilter: bloom.Estimate(n, 0.08), byte size rounded up to a power of two (at least 8), keys = big-endian sid */
void bloom_of(const std::vector<uint64_t> &sids, std::vector<uint8_t> &bits, uint64_t &m, uint64_t &k) {
    const double n = (double)sids.size(), ln2 = std::log(2.0);
    m = (uint64_t)std::ceil(-1.0 * n * std::log(0.08) / (ln2 * ln2));
    k = (uint64_t)std::ceil(ln2 * (double)m / n);
    uint64_t nb = 8; while (nb < (m + 7) / 8) nb *= 2;
    bits.assign(nb, 0);
    const uint64_t mask = nb * 8 - 1;
    for (uint64_t sid : sids) {
        uint8_t key[8]; for (int i = 0; i < 8; i++) key[i] = (uint8_t)(sid >> (56 - 8 * i));
        const uint64_t h0 = xxh64_8(key);
        key[7] = 0; /* Filter.hash: the second hash is of the key with its last byte cleared */
        const uint64_t h1 = xxh64_8(key);
        for (uint64_t i = 0; i < k; i++) { const uint64_t loc = (h0 + h1 * i) & mask; bits[loc >> 3] |= (uint8_t)(1u << (loc & 7)); }
    }
}

/* lib/encoding/int.go:66-212 Integer.Encoding: raw below three values, else zig-zag deltas as const-delta or Simple8b
 * (simple8b/encoding.go:350-473 EncodeAll; selectors 0/1 only when every remaining value is 1).  false where the reference falls
 * to zstd. */
bool int_block(const int64_t *v, size_t n, Wr &w) {
    auto zz = [](int64_t x) { return ((uint64_t)x << 1) ^ (uint64_t)(x >> 63); };
    if (n < 3) { w.u8(0x40); w.u32((uint32_t)(8 * n)); for (size_t i = 0; i < n; i++) w.u64(zz(v[i])); return true; }
    std::vector<uint64_t> d(n);
    d[0] = zz(v[0]);
    for (size_t i = 1; i < n; i++) d[i] = zz((int64_t)((uint64_t)v[i] - (uint64_t)v[i - 1]));
    bool is_const = true, is_s8b = true;
    for (size_t i = 1; i < n; i++) { if (i >= 2 && d[i] != d[i - 1]) is_const = false; if (d[i] > (1ull << 60) - 1) is_s8b = false; }
    auto uvarint = [&](uint64_t x) { while (x >= 0x80) { w.u8((uint32_t)(x & 0x7f) | 0x80); x >>= 7; } w.u8((uint32_t)x); };
    if (is_const) { w.u8(0x10); w.u64(d[0]); uvarint(d[1]); uvarint(n - 1); return true; }
    if (!is_s8b) return false;
    static const unsigned N[16] = {240, 120, 60, 30, 20, 15, 12, 10, 8, 7, 6, 5, 4, 3, 2, 1}, B[16] = {0, 0, 1, 2, 3, 4, 5, 6, 7, 8, 10, 12, 15, 20, 30, 60};
    std::vector<uint64_t> words;
    size_t ones_from = n; /* d[ones_from..] are all 1 */
    while (ones_from > 1 && d[ones_from - 1] == 1) ones_from--;
    for (size_t i = 1; i < n;) {
        int sel = 0;
        for (; sel < 16; sel++) {
            if (n - i < N[sel]) continue;
            bool ok = true;
            if (B[sel] == 0) ok = i >= ones_from;
            else for (unsigned k = 0; k < N[sel] && ok; k++) ok = d[i + k] <= (1ull << B[sel]) - 1;
            if (ok) break;
        }
        if (sel == 16) return false; /* unreachable: selector 15 packs any one value below 2^60 */
        uint64_t word = (uint64_t)sel << 60;
        if (B[sel]) for (unsigned k = 0; k < N[sel]; k++) word |= d[i + k] << (k * B[sel]);
        words.push_back(word); i += N[sel];
    }
    w.u8(0x20); w.u32((uint32_t)words.size() + 1); w.u32((uint32_t)n); w.u64(d[0]);
    for (uint64_t x : words) w.u64(x);
    return true;
}

} // namespace

int ogpu::tssp_build_tail(const TsspTailIn &in, std::vector<uint8_t> &out) {
    out.clear();
    Wr w{out};
    const uint32_t nc1 = in.n_cols1;
    const uint64_t meta_off = in.chunk_off[in.n_series];
    struct Item { uint64_t id; int64_t tmin, tmax; uint64_t off; uint32_t count, size; };
    std::vector<Item> items;
    std::vector<uint32_t> starts;
    std::vector<uint64_t> ids; std::vector<int64_t> rows, last_times;
    size_t block_begin = 0;
    int64_t file_tmin = INT64_MAX, file_tmax = INT64_MIN;
    Item cur{};
    auto close_block = [&]() { /* SwitchChunkMeta */
        for (uint32_t s : starts) w.u32(s);
        cur.size = (uint32_t)(out.size() - block_begin);
        items.push_back(cur);
        starts.clear(); block_begin = out.size(); cur = Item{};
    };
    for (uint32_t i = 0; i < in.n_series; i++) {
        const uint32_t g0 = in.seg_begin[i], nseg = in.seg_begin[i + 1] - g0;
        if (nseg == 0) continue; /* a series without rows has no chunk */
        const int64_t tmin = in.seg_tmin[g0], tmax = in.seg_tmax[g0 + nseg - 1]; /* ChunkMeta.MinMaxTime of a time-sorted chunk */
        if (cur.count == 0) { cur.id = in.sids[i]; cur.tmin = tmin; cur.tmax = tmax; cur.off = meta_off + block_begin; }
        cur.tmin = std::min(cur.tmin, tmin); cur.tmax = std::max(cur.tmax, tmax);
        file_tmin = std::min(file_tmin, tmin); file_tmax = std::max(file_tmax, tmax);
        starts.push_back((uint32_t)(out.size() - block_begin));
        uint32_t ncol = 0;
        for (uint32_t c = 0; c < nc1; c++) ncol += in.col_present[(size_t)i * nc1 + c];
        w.u64(in.sids[i]); w.i64((int64_t)in.chunk_off[i]); w.u32((uint32_t)(in.chunk_off[i + 1] - in.chunk_off[i])); w.u32(ncol); w.u32(nseg);
        for (uint32_t s = 0; s < nseg; s++) { w.i64(in.seg_tmin[g0 + s]); w.i64(in.seg_tmax[g0 + s]); }
        for (uint32_t c = 0; c < nc1; c++) {
            if (!in.col_present[(size_t)i * nc1 + c]) continue;
            const bool is_time = c + 1 == nc1;
            const std::string name = is_time ? "time" : in.col_names[c];
            const int type = is_time ? OG_TYPE_INT : in.col_types[c];
            w.u16((uint32_t)name.size()); w.bytes(name.data(), name.size()); w.u8((uint32_t)type);
            put_preagg(w, type, is_time, in.cells[(size_t)i * nc1 + c]);
            for (uint32_t s = 0; s < nseg; s++) { const size_t pi = (size_t)c * in.n_segments + g0 + s; w.i64((int64_t)in.page_off[pi]); w.u32(in.page_len[pi]); }
        }
        ids.push_back(in.sids[i]); rows.push_back(in.cells[(size_t)i * nc1 + nc1 - 1].count); last_times.push_back(tmax);
        cur.count++;
        if (out.size() - block_begin >= 256 * 1024 || cur.count >= 512) close_block(); /* needSwitchChunkMeta */
    }
    if (ids.empty()) { set_error("no series of the range holds rows: a TSSP file cannot be empty"); return OG_E_INVAL; }
    if (cur.count) close_block();
    const uint64_t index_size = out.size();
    for (const Item &m : items) { w.u64(m.id); w.i64(m.tmin); w.i64(m.tmax); w.i64((int64_t)m.off); w.u32(m.count); w.u32(m.size); }
    const uint64_t mi_size = out.size() - index_size;
    std::vector<uint8_t> bloom; uint64_t bloom_m, bloom_k;
    bloom_of(ids, bloom, bloom_m, bloom_k);
    w.bytes(bloom.data(), bloom.size());
    /* id-time: blocks of 2000 series, each [u32 count] then the sids, row counts and last times as length-prefixed integer blocks */
    const uint64_t idtime_begin = out.size();
    const uint32_t n = (uint32_t)ids.size(), per = 2000, blocks = (n + per - 1) / per;
    w.u32(n); w.u32(blocks);
    for (uint32_t b = 0; b < blocks; b++) {
        const uint32_t at = b * per, cnt = std::min(per, n - at);
        w.u32(cnt);
        const int64_t *arr[3] = {(const int64_t *)ids.data() + at, rows.data() + at, last_times.data() + at};
        for (int a = 0; a < 3; a++) {
            const size_t pos = out.size();
            w.u32(0);
            if (!int_block(arr[a], cnt, w)) {
                set_error("id-time section: the %s of series %u.. need the zstd integer form, which this writer does not produce; narrow the series range",
                          a == 0 ? "series ids" : a == 1 ? "row counts" : "last times", at);
                return OG_E_UNSUPPORTED;
            }
            const uint32_t sz = (uint32_t)(out.size() - pos - 4);
            for (int i = 0; i < 4; i++) out[pos + i] = (uint8_t)(sz >> (24 - 8 * i));
        }
    }
    const uint64_t idtime_size = out.size() - idtime_begin;
    const uint64_t trailer_off = meta_off + out.size();
    w.i64(16); w.i64((int64_t)(meta_off - 16)); w.i64((int64_t)index_size); w.i64((int64_t)mi_size); w.i64((int64_t)bloom.size()); w.i64((int64_t)idtime_size);
    w.i64((int64_t)ids.size()); w.u64(ids.front()); w.u64(ids.back()); w.i64(file_tmin); w.i64(file_tmax); w.i64((int64_t)items.size());
    w.u64(bloom_m); w.u64(bloom_k);
    /* ExtraData: time-store flag 1, compress flag 0, no chunk-meta header; its real length (10) in the upper half of the flags */
    w.u16(8);
    { const uint64_t flags = 1ull | (10ull << 32); for (int i = 0; i < 8; i++) w.u8((uint32_t)(flags >> (8 * i)) & 0xff); }
    w.u16(0);
    const size_t nl = strlen(in.measurement);
    w.u16((uint32_t)nl); w.bytes(in.measurement, nl);
    w.i64((int64_t)trailer_off);
    return OG_OK;
}
