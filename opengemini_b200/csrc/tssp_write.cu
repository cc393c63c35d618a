/*
 * tssp_write.cu — og_shard_write_tssp: an open shard -> the bytes of one TSSP file (version 2, attached layout, uncompressed
 * chunk metas).  Replaces, for data that is already on the device, MsBuilder.WriteData / Flush (engine/immutable/msbuilder.go:
 * 1248-1303,1355-1433), ChunkDataBuilder.EncodeChunk (chunkdata_builder_ts.go:37-82, chunkdata_builder.go:65-114) and the
 * pre-aggregation builders (pre_aggregation.go), whose inputs are decoded records: the pages are copied as they are, and only the
 * values pre-aggregation needs are pulled out of them.
 *
 *   1. k_preagg      a thread per (series, column) pulls the column's rows through ColIter / TimeIter and restates addValues of
 *                    IntegerPreAgg / FloatPreAgg / BooleanPreAgg / StringPreAgg / TimePreAgg; it also writes the byte length of
 *                    every slot of the column in file order: [4-byte CRC][page of segment 0][page of segment 1]...
 *   2. cub::DeviceScan over the slot lengths -> the offset of every CRC and page (first chunk at file offset 16)
 *   3. k_tssp_gather a warp per page copies the page to its place and computes its CRC32 from the bytes in flight.  CRC32 is
 *                    linear over GF(2): crc(A || B) = crc(A) * x^(8|B|) mod P  xor  crc(B).  So every lane multiplies the CRC of
 *                    its slice by x^(8 * bytes between the slice's end and the end of the COLUMN), and the xor of those products
 *                    over the lanes of all the column's pages is the column's CRC; no pass walks a column's bytes serially.
 *   4. k_tssp_crc_fold  a thread per (series, column) xors the column's page terms in segment order and stores the result
 *                    big-endian at the column's head.
 *   5. the host gets the pre-agg cells, the chunk offsets and the new page directory and builds everything behind the chunks
 *      (tssp.cpp tssp_build_tail).  og_tssp_image_export copies the chunk region out in one transfer.
 *
 * Only pages the directory references are copied: a merged shard's rewritten source pages stay behind.
 */
#include <cub/device/device_scan.cuh>

#include <chrono>
#include <cstring>
#include <memory>
#include <vector>

#include "decode.cuh"
#include "internal.h"
#include "tssp_write.h"

using namespace ogpu;

namespace {

constexpr uint32_t CRC_POLY = 0xedb88320u;       /* IEEE 802.3, reflected: Go hash/crc32.ChecksumIEEE, zlib crc32 */
constexpr uint64_t FILE_SIZE_LIMIT = 8ull << 30; /* lib/util/util.go:83 DefaultFileSizeLimit */
constexpr uint32_t SEGMENT_LIMIT = 65535;        /* engine/immutable/config.go:25 maxSegmentLimit */
constexpr uint64_t MAX_F64 = 0x7fefffffffffffffull, NEG_MAX_F64 = 0xffefffffffffffffull;

struct WriteP { /* the shard's directory and the range being written */
    const uint8_t *data;
    const uint64_t *page_off; const uint32_t *page_len; /* [(n_columns + 1) * n_segments], time last */
    const uint32_t *seg_series, *seg_rows, *series_seg_begin;
    uint32_t n_segments, n_cols1;
    uint32_t series0, n_series; /* series [series0, series0 + n_series) */
    uint32_t seg0, n_seg;       /* their segments [seg0, seg0 + n_seg) */
};

/* slots of the written range in file order: per series, per column, one CRC slot then one slot per segment */
__device__ __forceinline__ uint64_t column_slot(const WriteP &w, uint32_t series, uint32_t col, uint32_t *n_seg) {
    const uint32_t b = w.series_seg_begin[series], n = w.series_seg_begin[series + 1] - b;
    *n_seg = n;
    return (uint64_t)(series - w.series0) * w.n_cols1 + (uint64_t)(b - w.seg0) * w.n_cols1 + (uint64_t)col * (1 + n);
}

__device__ __forceinline__ void report(int *err, int code, uint32_t seg) {
    if (atomicCAS(err, 0, code) == 0) err[1] = (int)seg;
}

/* addValues of one field type over the rows of one segment.  TYPE is the column type; the codec switch stays inside ColIter. */
template <int TYPE> __device__ __forceinline__ void preagg_segment(ColIter &it, TimeIter &tm, uint32_t rows, PreAggCell &a) {
    if constexpr (TYPE == OG_TYPE_BOOL) {
        /* BooleanPreAgg.addValues walks the VALUES and indexes times by the value index (pre_aggregation.go:749-765): with nulls
         * the recorded time is that of row j of the segment, not of the row that holds the j-th value.  Kept as it is. */
        for (uint32_t r = 0; r < rows; r++) {
            uint64_t v;
            if (!it.next(v)) continue;
            const int64_t t = tm.next(); /* pulled once per value: the time of row j */
            if ((int64_t)a.minv > (int64_t)v) { a.minv = v; a.mint = t; }
            if ((int64_t)a.maxv < (int64_t)v) { a.maxv = v; a.maxt = t; }
        }
    } else for (uint32_t r = 0; r < rows; r++) {
        const int64_t t = tm.next();
        uint64_t v;
        if (!it.next(v)) continue;
        if constexpr (TYPE == OG_TYPE_FLOAT) { /* strict compares: the first occurrence wins and a NaN never replaces anything */
            const double f = __longlong_as_double((long long)v);
            if (__longlong_as_double((long long)a.minv) > f) { a.minv = v; a.mint = t; }
            if (__longlong_as_double((long long)a.maxv) < f) { a.maxv = v; a.maxt = t; }
            a.sum = (uint64_t)__double_as_longlong(__dadd_rn(__longlong_as_double((long long)a.sum), f)); /* sumV += v in row order */
        } else {
            if ((int64_t)a.minv > (int64_t)v) { a.minv = v; a.mint = t; }
            if ((int64_t)a.maxv < (int64_t)v) { a.maxv = v; a.maxt = t; }
            a.sum += v; /* wraps, as int64 does */
        }
    }
}

/* thread per (series, column): the column's pre-aggregation over the rows of the chunk, and its slot lengths */
__global__ void k_preagg(WriteP w, const int32_t *types, PreAggCell *cells, uint8_t *col_state /* 0 absent, 1 present, 2 in some segments only */,
                         uint64_t *slot_len, int *err) {
    const uint64_t id = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (id >= (uint64_t)w.n_series * w.n_cols1) return;
    const uint32_t series = w.series0 + (uint32_t)(id / w.n_cols1), col = (uint32_t)(id % w.n_cols1);
    uint32_t n;
    const uint64_t slot = column_slot(w, series, col, &n);
    const uint32_t g0 = w.series_seg_begin[series];
    const bool is_time = col + 1 == w.n_cols1;
    const int type = is_time ? OG_TYPE_INT : types[col];
    PreAggCell a;
    a.mint = a.maxt = 0; a.sum = 0; a.count = 0;
    if (type == OG_TYPE_FLOAT) { a.minv = MAX_F64; a.maxv = NEG_MAX_F64; }
    else if (type == OG_TYPE_BOOL) { a.minv = 2; a.maxv = (uint64_t)-1ll; }
    else { a.minv = (uint64_t)INT64_MAX; a.maxv = (uint64_t)INT64_MIN; }
    uint32_t present = 0;
    for (uint32_t j = 0; j < n; j++) {
        const uint32_t g = g0 + j, rows = w.seg_rows[g];
        const size_t pi = (size_t)col * w.n_segments + g;
        const uint32_t len = w.page_len[pi];
        slot_len[slot + 1 + j] = len;
        if (is_time) { a.count += rows; present++; continue; } /* TimePreAgg: the row count */
        if (len == 0) continue;
        present++;
        ColIter it;
        it.init(w.data + w.page_off[pi], len, type, rows);
        if (it.err != D_OK) { report(err, it.err, g); continue; }
        a.count += it.h.rows - it.h.nil_count;
        if (type == OG_TYPE_STRING || it.kind == ColIter::K_ABSENT) continue; /* strings: the count comes from the validity bitmap */
        const size_t ti = (size_t)(w.n_cols1 - 1) * w.n_segments + g;
        TimeDesc td;
        const int rc = parse_time_page(w.data + w.page_off[ti], w.page_len[ti], td);
        if (rc != D_OK) { report(err, rc, g); continue; }
        TimeIter tm; tm.init(td);
        if (type == OG_TYPE_FLOAT) preagg_segment<OG_TYPE_FLOAT>(it, tm, rows, a);
        else if (type == OG_TYPE_INT) preagg_segment<OG_TYPE_INT>(it, tm, rows, a);
        else preagg_segment<OG_TYPE_BOOL>(it, tm, rows, a);
        it.finish();
        if (type != OG_TYPE_BOOL) tm.finish(); /* the bool builder does not walk the time page to its end */
        if (it.err != D_OK) report(err, it.err, g);
        else if (tm.err != D_OK) report(err, tm.err, g);
    }
    slot_len[slot] = present ? 4 : 0;
    cells[id] = a;
    col_state[id] = present == 0 ? 0 : present == n ? 1 : 2;
}

/* ---- CRC32 arithmetic in GF(2)[x] mod P, reflected bit order: bit 31 is x^0 ---- */
struct CrcPow { uint32_t p[32]; }; /* x^(2^k) mod P */

__host__ __device__ inline uint32_t crc_mul(uint32_t a, uint32_t b) { /* a * b mod P */
    uint32_t p = 0;
    for (int i = 31; i >= 0; i--) {
        p ^= b & (0u - ((a >> i) & 1u));
        b = (b >> 1) ^ (CRC_POLY & (0u - (b & 1u)));
    }
    return p;
}
__host__ __device__ inline uint32_t crc_x_pow_bytes(const CrcPow &t, uint64_t n_bytes) { /* x^(8 n) mod P */
    uint32_t p = 0x80000000u;
    for (uint32_t k = 3; n_bytes; n_bytes >>= 1, k++) if (n_bytes & 1) p = crc_mul(t.p[k & 31], p); /* x has order 2^32 - 1: x^(2^32) = x */
    return p;
}

constexpr int GATHER_THREADS = 256;

/* warp per page of the written range */
__global__ void __launch_bounds__(GATHER_THREADS) k_tssp_gather(WriteP w, const uint64_t *slot_off, CrcPow pw, uint8_t *out,
                                                                uint64_t *new_page_off, uint32_t *page_term) {
    __shared__ uint32_t T[4][256]; /* slice-by-4 tables */
    {
        uint32_t c = threadIdx.x;
        for (int k = 0; k < 8; k++) c = (c >> 1) ^ (CRC_POLY & (0u - (c & 1u)));
        T[0][threadIdx.x] = c;
        __syncthreads();
        for (int t = 1; t < 4; t++) { c = (c >> 8) ^ T[0][c & 0xff]; T[t][threadIdx.x] = c; }
        __syncthreads();
    }
    const uint64_t page = ((uint64_t)blockIdx.x * GATHER_THREADS + threadIdx.x) >> 5;
    const uint32_t lane = threadIdx.x & 31;
    if (page >= (uint64_t)w.n_cols1 * w.n_seg) return;
    const uint32_t col = (uint32_t)(page / w.n_seg), g = w.seg0 + (uint32_t)(page % w.n_seg);
    const uint32_t series = w.seg_series[g];
    uint32_t n;
    const uint64_t cslot = column_slot(w, series, col, &n);
    const uint64_t off = slot_off[cslot + 1 + (g - w.series_seg_begin[series])], col_end = slot_off[cslot + 1 + n];
    const size_t pi = (size_t)col * w.n_segments + g;
    const uint32_t len = w.page_len[pi];
    if (lane == 0) new_page_off[page] = 16 + off;
    if (len == 0) { if (lane == 0) page_term[page] = 0; return; }
    const uint8_t *src = w.data + w.page_off[pi];
    uint8_t *dst = out + off;
    /* each lane owns a contiguous slice, a multiple of 16 bytes long */
    const uint32_t slice = (((len + 31) >> 5) + 15) & ~15u;
    const uint32_t lo = min(lane * slice, len), hi = min(lo + slice, len);
    uint32_t crc = 0xffffffffu, i = lo;
    for (; i < hi && ((uintptr_t)(dst + i) & 15); i++) { const uint8_t b = __ldg(src + i); dst[i] = b; crc = T[0][(crc ^ b) & 0xff] ^ (crc >> 8); }
    if (i + 16 <= hi) { /* 16-byte stores; the source is read in aligned 8-byte words and shifted into place */
        const uintptr_t sa = (uintptr_t)(src + i);
        const uint64_t *q = (const uint64_t *)(sa & ~(uintptr_t)7);
        const unsigned sh = (unsigned)(sa & 7) * 8;
        uint64_t w0 = __ldg(q);
        for (; i + 16 <= hi; i += 16, q += 2) {
            const uint64_t w1 = __ldg(q + 1);
            uint64_t a = w0, b = w1;
            if (sh) { const uint64_t w2 = __ldg(q + 2); a = (w0 >> sh) | (w1 << (64 - sh)); b = (w1 >> sh) | (w2 << (64 - sh)); w0 = w2; }
            else w0 = __ldg(q + 2); /* at most 23 bytes past the slice: inside the 1024 bytes that follow every shard's data */
            *(uint4 *)(dst + i) = make_uint4((uint32_t)a, (uint32_t)(a >> 32), (uint32_t)b, (uint32_t)(b >> 32));
            const uint32_t word[4] = {(uint32_t)a, (uint32_t)(a >> 32), (uint32_t)b, (uint32_t)(b >> 32)};
#pragma unroll
            for (int k = 0; k < 4; k++) {
                crc ^= word[k];
                crc = T[3][crc & 0xff] ^ T[2][(crc >> 8) & 0xff] ^ T[1][(crc >> 16) & 0xff] ^ T[0][crc >> 24];
            }
        }
    }
    for (; i < hi; i++) { const uint8_t b = __ldg(src + i); dst[i] = b; crc = T[0][(crc ^ b) & 0xff] ^ (crc >> 8); }
    crc = ~crc; /* an empty slice yields 0, the CRC of nothing */
    uint32_t term = crc_mul(crc_x_pow_bytes(pw, col_end - (off + hi)), crc);
    term = __reduce_xor_sync(0xffffffffu, term);
    if (lane == 0) page_term[page] = term;
}

/* thread per (series, column): CRC of the column = xor of its pages' terms; stored big-endian in front of the pages */
__global__ void k_tssp_crc_fold(WriteP w, const uint64_t *slot_off, const uint32_t *page_term, const uint8_t *col_state, uint8_t *out, uint64_t *chunk_off) {
    const uint64_t id = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (id >= (uint64_t)w.n_series * w.n_cols1) return;
    const uint32_t series = w.series0 + (uint32_t)(id / w.n_cols1), col = (uint32_t)(id % w.n_cols1);
    uint32_t n;
    const uint64_t slot = column_slot(w, series, col, &n);
    if (col == 0) chunk_off[series - w.series0] = 16 + slot_off[slot];
    if (!col_state[id]) return;
    const uint32_t *t = page_term + (size_t)col * w.n_seg + (w.series_seg_begin[series] - w.seg0);
    uint32_t crc = 0;
    for (uint32_t j = 0; j < n; j++) crc ^= t[j];
    uint8_t *p = out + slot_off[slot];
    p[0] = (uint8_t)(crc >> 24); p[1] = (uint8_t)(crc >> 16); p[2] = (uint8_t)(crc >> 8); p[3] = (uint8_t)crc;
}

} // namespace

struct og_tssp_image {
    int device = 0;
    uint8_t *d_chunks = nullptr; uint64_t chunk_bytes = 0; /* file bytes [16, 16 + chunk_bytes), on the device */
    std::vector<uint8_t> tail;                             /* everything behind the chunks */
    double phase_ms[4] = {0, 0, 0, 0};
    ~og_tssp_image() { cudaSetDevice(device); dev_free(d_chunks); }
};

extern "C" {

OG_API void og_tssp_image_free(og_tssp_image *f) { delete f; }

OG_API int og_shard_write_tssp(og_shard *s, const og_tssp_write_desc *d, og_tssp_image **out) {
    if (!s || !d || !out) { set_error("null argument"); return OG_E_INVAL; }
    *out = nullptr;
    if (!d->measurement || strlen(d->measurement) > 0xffff) { set_error("measurement name missing or longer than 65535 bytes"); return OG_E_INVAL; }
    if (d->flags) { set_error("unknown flags 0x%x", d->flags); return OG_E_INVAL; }
    CU(cudaSetDevice(s->device));
    uint32_t sb = d->series_begin, se = d->series_end;
    if (sb == 0 && se == 0) se = s->n_series;
    if (sb >= se || se > s->n_series) { set_error("empty or out-of-range series range [%u, %u) of %u series", sb, se, s->n_series); return OG_E_INVAL; }
    const std::vector<uint32_t> &ssb = s->h_series_seg_begin;
    for (uint32_t i = sb; i < se; i++) {
        if (s->sids[i] == 0 || (i > sb && s->sids[i] <= s->sids[i - 1])) { /* msbuilder.go:1252-1256 */
            set_error("series ids must be non-zero and strictly ascending (series %u has id %llu)", i, (unsigned long long)s->sids[i]); return OG_E_INVAL;
        }
        if (ssb[i + 1] - ssb[i] > SEGMENT_LIMIT) {
            set_error("series %u has %u segments; a chunk holds at most %u", i, ssb[i + 1] - ssb[i], SEGMENT_LIMIT); return OG_E_UNSUPPORTED;
        }
    }
    WriteP w;
    w.data = s->d_data; w.page_off = s->d_page_off; w.page_len = s->d_page_len; w.seg_series = s->d_seg_series; w.seg_rows = s->d_seg_rows;
    w.series_seg_begin = s->d_series_seg_begin; w.n_segments = s->n_segments; w.n_cols1 = s->n_columns + 1;
    w.series0 = sb; w.n_series = se - sb; w.seg0 = ssb[sb]; w.n_seg = ssb[se] - ssb[sb];
    if (w.n_seg == 0) { set_error("no series of the range holds rows: a TSSP file cannot be empty"); return OG_E_INVAL; }
    const size_t n_cells = (size_t)w.n_series * w.n_cols1, n_pages = (size_t)w.n_cols1 * w.n_seg, n_slots = n_cells + n_pages;
    if (n_slots + 1 > 0x7fffffffull) { set_error("%zu pages and columns in one file; narrow the series range", n_slots); return OG_E_UNSUPPORTED; }

    std::unique_ptr<og_tssp_image> img(new og_tssp_image);
    img->device = s->device;
    Scratch fr;
    int rc;
    int32_t *d_types; PreAggCell *d_cells; uint8_t *d_state; uint64_t *d_slot_len, *d_slot_off, *d_new_off, *d_chunk_off; uint32_t *d_term; int *d_err;
    if ((rc = fr.get(&d_types, s->n_columns)) || (rc = fr.get(&d_cells, n_cells)) || (rc = fr.get(&d_state, n_cells)) ||
        (rc = fr.get(&d_slot_len, n_slots + 1)) || (rc = fr.get(&d_slot_off, n_slots + 1)) || (rc = fr.get(&d_new_off, n_pages)) ||
        (rc = fr.get(&d_chunk_off, (size_t)w.n_series)) || (rc = fr.get(&d_term, n_pages)) || (rc = fr.get(&d_err, 2))) return rc;
    CU(cudaMemcpy(d_types, s->col_types.data(), s->n_columns * sizeof(int32_t), cudaMemcpyHostToDevice));
    CU(cudaMemset(d_err, 0, 8));
    CU(cudaMemset(d_slot_len + n_slots, 0, 8)); /* the scan's last output is then the size of the chunk region */

    /* ---- phase 0: pre-aggregation and slot lengths ---- */
    auto t0 = std::chrono::steady_clock::now();
    k_preagg<<<(unsigned)((n_cells + 127) / 128), 128>>>(w, d_types, d_cells, d_state, d_slot_len, d_err);
    CU(cudaGetLastError());
    int err[2];
    CU(cudaMemcpy(err, d_err, 8, cudaMemcpyDeviceToHost));
    if (err[0]) {
        set_error("segment %d failed to decode (device code %d)", err[1], err[0]);
        return map_dev_err(err[0]);
    }
    img->phase_ms[0] = ms_since(t0);

    /* ---- phase 1: layout, gather, CRC ---- */
    t0 = std::chrono::steady_clock::now();
    {
        void *tmp = nullptr; size_t tb = 0;
        CU(cub::DeviceScan::ExclusiveSum(nullptr, tb, d_slot_len, d_slot_off, (int)(n_slots + 1)));
        if ((rc = fr.get((uint8_t **)&tmp, tb))) return rc;
        CU(cub::DeviceScan::ExclusiveSum(tmp, tb, d_slot_len, d_slot_off, (int)(n_slots + 1)));
    }
    CU(cudaMemcpy(&img->chunk_bytes, d_slot_off + n_slots, 8, cudaMemcpyDeviceToHost));
    if (16 + img->chunk_bytes > FILE_SIZE_LIMIT) {
        set_error("the chunks of series [%u, %u) take %llu bytes; a file holds at most %llu: narrow the series range", sb, se,
                  (unsigned long long)img->chunk_bytes, (unsigned long long)FILE_SIZE_LIMIT);
        return OG_E_UNSUPPORTED;
    }
    if ((rc = dalloc(&img->d_chunks, (size_t)img->chunk_bytes))) return rc;
    static const CrcPow pw = [] { CrcPow t; uint32_t p = 1u << 30; t.p[0] = p; for (int k = 1; k < 32; k++) t.p[k] = p = crc_mul(p, p); return t; }();
    k_tssp_gather<<<(unsigned)((n_pages * 32 + GATHER_THREADS - 1) / GATHER_THREADS), GATHER_THREADS>>>(w, d_slot_off, pw, img->d_chunks, d_new_off, d_term);
    CU(cudaGetLastError());
    k_tssp_crc_fold<<<(unsigned)((n_cells + 127) / 128), 128>>>(w, d_slot_off, d_term, d_state, img->d_chunks, d_chunk_off);
    CU(cudaGetLastError());
    CU(cudaDeviceSynchronize());
    img->phase_ms[1] = ms_since(t0);

    /* ---- phase 2: metadata to the host ---- */
    t0 = std::chrono::steady_clock::now();
    std::vector<PreAggCell> cells(n_cells); std::vector<uint8_t> state(n_cells);
    std::vector<uint64_t> chunk_off((size_t)w.n_series + 1), new_off(n_pages); std::vector<uint32_t> page_len(n_pages);
    std::vector<int64_t> tmin(w.n_seg), tmax(w.n_seg);
    CU(cudaMemcpy(cells.data(), d_cells, n_cells * sizeof(PreAggCell), cudaMemcpyDeviceToHost));
    CU(cudaMemcpy(state.data(), d_state, n_cells, cudaMemcpyDeviceToHost));
    CU(cudaMemcpy(chunk_off.data(), d_chunk_off, (size_t)w.n_series * 8, cudaMemcpyDeviceToHost));
    CU(cudaMemcpy(new_off.data(), d_new_off, n_pages * 8, cudaMemcpyDeviceToHost));
    CU(cudaMemcpy2D(page_len.data(), (size_t)w.n_seg * 4, s->d_page_len + w.seg0, (size_t)s->n_segments * 4, (size_t)w.n_seg * 4, w.n_cols1, cudaMemcpyDeviceToHost));
    CU(cudaMemcpy(tmin.data(), s->d_tmin + w.seg0, (size_t)w.n_seg * 8, cudaMemcpyDeviceToHost));
    CU(cudaMemcpy(tmax.data(), s->d_tmax + w.seg0, (size_t)w.n_seg * 8, cudaMemcpyDeviceToHost));
    chunk_off[w.n_series] = 16 + img->chunk_bytes;
    img->phase_ms[2] = ms_since(t0);

    /* ---- phase 3: everything behind the chunks ---- */
    t0 = std::chrono::steady_clock::now();
    for (size_t i = 0; i < n_cells; i++)
        if (state[i] == 2) {
            const uint32_t series = sb + (uint32_t)(i / w.n_cols1), col = (uint32_t)(i % w.n_cols1);
            set_error("series %u holds column %s in some of its segments only: a chunk lists a column for every segment or not at all", series, s->col_names[col].c_str());
            return OG_E_UNSUPPORTED;
        }
    std::vector<uint32_t> seg_begin((size_t)w.n_series + 1);
    for (uint32_t i = 0; i <= w.n_series; i++) seg_begin[i] = ssb[sb + i] - w.seg0;
    TsspTailIn in;
    in.measurement = d->measurement; in.n_series = w.n_series; in.n_segments = w.n_seg; in.n_cols1 = w.n_cols1;
    in.sids = s->sids.data() + sb; in.seg_begin = seg_begin.data(); in.seg_tmin = tmin.data(); in.seg_tmax = tmax.data();
    in.col_names = s->col_names.data(); in.col_types = s->col_types.data(); in.cells = cells.data(); in.col_present = state.data();
    in.chunk_off = chunk_off.data(); in.page_off = new_off.data(); in.page_len = page_len.data();
    if ((rc = tssp_build_tail(in, img->tail))) return rc;
    if (16 + img->chunk_bytes + img->tail.size() > FILE_SIZE_LIMIT) {
        set_error("the file of series [%u, %u) would take %llu bytes; a file holds at most %llu: narrow the series range", sb, se,
                  (unsigned long long)(16 + img->chunk_bytes + img->tail.size()), (unsigned long long)FILE_SIZE_LIMIT);
        return OG_E_UNSUPPORTED;
    }
    img->phase_ms[3] = ms_since(t0);
    *out = img.release();
    return OG_OK;
}

OG_API int og_tssp_image_size(const og_tssp_image *f, uint64_t *bytes) {
    if (!f || !bytes) { set_error("null argument"); return OG_E_INVAL; }
    *bytes = 16 + f->chunk_bytes + f->tail.size();
    return OG_OK;
}

OG_API int og_tssp_image_export(const og_tssp_image *f, uint8_t *host) {
    if (!f || !host) { set_error("null argument"); return OG_E_INVAL; }
    CU(cudaSetDevice(f->device));
    memcpy(host, "53ac2021", 8); /* tableMagic, then the version (engine/immutable/table.go:24-28) */
    for (int i = 0; i < 8; i++) host[8 + i] = i == 7 ? 2 : 0;
    CU(cudaMemcpy(host + 16, f->d_chunks, f->chunk_bytes, cudaMemcpyDeviceToHost));
    memcpy(host + 16 + f->chunk_bytes, f->tail.data(), f->tail.size());
    return OG_OK;
}

OG_API int og_tssp_image_timing(const og_tssp_image *f, double phase_ms[4]) {
    if (!f || !phase_ms) { set_error("null argument"); return OG_E_INVAL; }
    memcpy(phase_ms, f->phase_ms, sizeof f->phase_ms);
    return OG_OK;
}

} // extern "C"
