/*
 * internal.h — host-side handle layouts and kernel parameter blocks shared by the .cu files of libogpu.so.
 */
#pragma once
#include <cuda_runtime.h>

#include <chrono>
#include <cstdint>
#include <memory>
#include <string>
#include <mutex>
#include <vector>

#include "../../include/ogpu.h"

#define OG_MAX_CALLS 8
#define OG_MAX_FILTER 16
#define OG_MAX_COLS 8 /* distinct field columns one query may touch */

namespace ogpu {

void set_error(const char *fmt, ...);
int cuda_fail(cudaError_t e, const char *what, const char *file, int line);
int ensure_device(); /* bind the calling thread to the library's device (og_init(0) on first use) */
int map_dev_err(int device_code); /* a device decode code (decode.cuh D_*) as the OG_E_* status a call returns */

inline double ms_since(std::chrono::steady_clock::time_point t0) {
    return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
}

/* two events that time work on one stream: start() creates and records the first, stop() records the second, ms() is the time
 * between them once the stop event has completed */
struct EventTimer {
    cudaStream_t stream;
    cudaEvent_t ev[2] = {nullptr, nullptr};
    explicit EventTimer(cudaStream_t st = 0) : stream(st) {}
    EventTimer(const EventTimer &) = delete;
    EventTimer &operator=(const EventTimer &) = delete;
    ~EventTimer() { for (cudaEvent_t e : ev) if (e) cudaEventDestroy(e); }
    cudaError_t start() {
        for (cudaEvent_t &e : ev) { const cudaError_t r = cudaEventCreate(&e); if (r != cudaSuccess) return r; }
        return cudaEventRecord(ev[0], stream);
    }
    cudaError_t stop() { return cudaEventRecord(ev[1], stream); }
    cudaError_t ms(double *out) const { float m = 0; const cudaError_t e = cudaEventElapsedTime(&m, ev[0], ev[1]); *out = m; return e; }
};

/* api.cu: the steps of opening a shard */
int check_desc(const og_shard_desc *d);
int alloc_dir(og_shard *s);
int upload_dir(og_shard *s, const uint32_t *series_seg_begin, const int64_t *seg_tmin, const int64_t *seg_tmax, const uint64_t *page_off,
               const uint32_t *page_len, const uint64_t *sids);
int shard_finalize(og_shard *s, bool scan_snappy);
/* encode.cu: og_encode_pages; nan_raw: see encode_float_page */
int encode_pages(int32_t type, int32_t is_time, const void *d_values, const uint8_t *d_valid, const uint32_t *d_rows, uint32_t n_segments,
                 uint32_t rps, uint8_t *d_out, uint64_t out_cap, uint64_t *d_page_off, uint32_t *d_page_len, uint64_t *total_bytes_out,
                 bool nan_raw);

/* Device memory comes from the device's stream-ordered pool (cudaMallocAsync on the legacy stream) with its release threshold
 * raised at og_init: shards and queries that are opened and closed in a loop get their buffers back from the pool instead of
 * paying cudaMalloc/cudaFree (tens of ms per GB-sized buffer) every time.  A buffer is owned by a handle (og_shard, og_query,
 * og_downsampled, og_tssp_image, og_merge_state: their destructors free it) or by a Scratch for the length of one call.  The
 * release goes to the legacy stream, which orders it after legacy-stream work; a buffer used on another stream is released
 * only after that stream has been synchronised (~og_query and a Scratch bound to the stream do it). */
inline cudaError_t dev_malloc(void **p, size_t bytes) { return cudaMallocAsync(p, bytes ? bytes : 1, (cudaStream_t)0); }
inline void dev_free(void *p) { if (p) cudaFreeAsync(p, (cudaStream_t)0); }
template <class... T> void dev_free_all(T *...p) { (dev_free((void *)p), ...); }
/* free device memory as a budget sees it: what the driver reports plus what the pool holds but does not use */
cudaError_t dev_mem_info(size_t *free_b, size_t *total_b);
#define CU(call) do { cudaError_t e__ = (call); if (e__ != cudaSuccess) return ::ogpu::cuda_fail(e__, #call, __FILE__, __LINE__); } while (0)

/* n elements of T (at least one byte); OG_E_NOMEM or OG_E_CUDA with the error text set */
template <class T> int dalloc(T **p, size_t n) {
    *p = nullptr;
    if (n == 0) n = 1;
    cudaError_t e = dev_malloc((void **)p, n * sizeof(T));
    if (e != cudaSuccess) { set_error("cudaMalloc(%zu bytes) failed: %s", n * sizeof(T), cudaGetErrorString(e)); return e == cudaErrorMemoryAllocation ? OG_E_NOMEM : OG_E_CUDA; }
    return OG_OK;
}

/* device buffers freed together when the Scratch goes out of scope; bound to a stream (not the legacy one), it synchronises
 * that stream first, so no kernel still enqueued there reads a buffer that went back to the pool */
struct Scratch {
    cudaStream_t stream = nullptr;
    std::vector<void *> bufs;
    Scratch() = default;
    explicit Scratch(cudaStream_t st) : stream(st) {}
    Scratch(const Scratch &) = delete;
    Scratch &operator=(const Scratch &) = delete;
    ~Scratch() {
        if (stream && !bufs.empty()) cudaStreamSynchronize(stream);
        for (void *p : bufs) dev_free(p);
    }
    template <class T> int get(T **p, size_t n) { int rc = dalloc(p, n); if (rc == OG_OK) bufs.push_back(*p); return rc; }
};

/* the live queries of a shard: og_query_create counts up, ~og_query down, a rewrite of the shard (rewrite_shard, span_pass.h)
 * holds `mu` throughout.  Shared by the shard and its queries, so a query destroyed after its shard was closed still finds it. */
struct LiveQueries { std::mutex mu; uint32_t n = 0; };

/* everything that describes a shard's rows and where they live: a rewrite builds a new one and install_state (span_pass.h) swaps
 * it in whole */
struct ShardState {
    int device = 0;
    uint8_t *d_data = nullptr; uint64_t data_len = 0; bool owns_data = true;
    uint32_t n_series = 0, n_segments = 0, n_columns = 0;
    uint32_t max_seg_rows = 0;
    uint64_t irregular_time_pages = 0; /* time pages that are neither const-delta nor one-row (Simple8b / raw times) */
    uint64_t n_rows = 0, page_bytes = 0;
    uint64_t snappy_pages = 0, snappy_bytes_in = 0, snappy_bytes_out = 0; /* Snappy pages transcoded to raw at open */
    og_merge_info merge{1, 0, 0, 0, 0, 0, 0, 0, 0, 0}; /* og_shard_open_files (merge.cu); one file and zeros otherwise */
    bool rows_merged = false; /* some open or append re-encoded a span: the Snappy counters were dropped with the file set's region */
    int64_t tmin = 0, tmax = 0;
    std::vector<uint64_t> sids;
    std::vector<int32_t> col_types;
    std::vector<std::string> col_names;
    std::vector<uint32_t> h_series_seg_begin; /* always mirrored on host (n_series+1) */
    /* device directory (SoA) */
    uint32_t *d_series_seg_begin = nullptr; /* [n_series+1] */
    uint32_t *d_seg_series = nullptr;       /* [n_segments] */
    uint32_t *d_seg_rows = nullptr;         /* [n_segments] rows per segment (from the time page) */
    int64_t *d_tmin = nullptr, *d_tmax = nullptr; /* [n_segments] */
    uint64_t *d_page_off = nullptr;         /* [(n_columns+1) * n_segments], time column last */
    uint32_t *d_page_len = nullptr;
    uint64_t *d_sids = nullptr;
};

} // namespace ogpu

struct og_shard : ogpu::ShardState {
    /* materialise scratch for og_decode_segment (host pinned + device) */
    void *h_seg_buf = nullptr; size_t h_seg_buf_bytes = 0;
    void *d_seg_buf = nullptr; size_t d_seg_buf_bytes = 0;
    std::vector<og_colval_view> seg_views;
    /* lane-interleaved, length-binned stream copy per column for the fused Gorilla kernel (fused_il.cuh), built on first use */
    struct IlCol { int state = 0; /* 0 not built, 1 ready, -1 no eligible segment, -2 not enough device memory (general kernel serves the column) */
                   uint32_t *words = nullptr; uint64_t *grp_off = nullptr; uint32_t *grp_rows = nullptr, *grp_col = nullptr;
                   uint32_t *lane_seg = nullptr, *lane_rows = nullptr, *lane_series = nullptr; uint16_t *lane_win = nullptr; int64_t *lane_t0 = nullptr; uint64_t *lane_dt = nullptr;
                   uint32_t *gen_list = nullptr; std::vector<uint32_t> gen_host; /* segments the fused kernel does not take (ascending), device + host */
                   uint32_t n_groups = 0, J = 0; /* J != 0: regular shard, lane groups share a segment index */
                   bool aligned = false; /* regular shard whose segment index j has one [seg_tmin, seg_tmax] in every series of a binning domain */
                   uint32_t n_super = 1, cols_per_super = 0; std::vector<uint32_t> super_grp_first; /* [n_super+1] first lane group of each block of OG_IL_SUPER series */
                   uint64_t n_words = 0, n_packed = 0; /* words of the copy; segments stored as packed XOR deltas */ double build_ms = 0; };
    std::vector<IlCol> il; /* [n_columns] */
    std::mutex il_mu;      /* queries of one shard may be planned from different threads: the build is serialised */
    std::shared_ptr<ogpu::LiveQueries> live = std::make_shared<ogpu::LiveQueries>();
    /* every interleaved copy freed, one unbuilt entry per column left: a rewrite of the shard drops the copies of the old layout,
     * and the first query that wants one builds it again */
    void reset_il() {
        std::lock_guard<std::mutex> lock(il_mu);
        for (IlCol &c : il)
            ogpu::dev_free_all(c.words, c.grp_off, c.grp_rows, c.grp_col, c.lane_seg, c.lane_rows, c.lane_series, c.lane_win, c.lane_t0, c.lane_dt, c.gen_list);
        il.assign(n_columns, IlCol{});
    }
    ~og_shard() {
        using ogpu::dev_free_all;
        if (owns_data) dev_free_all(d_data);
        dev_free_all(d_series_seg_begin, d_seg_series, d_seg_rows, d_tmin, d_tmax, d_page_off, d_page_len, d_sids, d_seg_buf);
        if (h_seg_buf) cudaFreeHost(h_seg_buf);
        reset_il();
    }
};

namespace ogpu {

struct CallP { int32_t func, col_slot, type, out_type; };
struct FilterP { int32_t kind, col_slot, op, type, const_is_float; double fval; int64_t ival; };

/* per-call cell/edge/dense array triple */
struct Tri { uint64_t *val; int64_t *tim; uint8_t *ok; };

struct QueryP { /* passed by value to kernels */
    int64_t tmin, tmax, start, interval; /* interval = window length (end-start of Window()); >0 always on device */
    uint32_t n_buckets, n_calls, n_filter, n_cols;
    int32_t multi; /* callCount > 1 */
    CallP calls[OG_MAX_CALLS];
    FilterP filter[OG_MAX_FILTER];
    int32_t col_index[OG_MAX_COLS]; /* shard column of each slot */
    int32_t col_type[OG_MAX_COLS];
};

} // namespace ogpu

struct og_query {
    og_shard *sh = nullptr;
    std::shared_ptr<ogpu::LiveQueries> live; /* the shard's live-query count, which this query is part of */
    og_query_desc desc{};
    std::vector<og_call> calls;
    std::vector<og_filter_item> filter;
    std::vector<uint32_t> series_group;
    cudaStream_t stream = nullptr;
    cudaEvent_t ev0 = nullptr, ev1 = nullptr;
    ogpu::QueryP qp{};
    uint32_t n_groups = 0;
    bool ran = false; volatile int aborted = 0;
    /* dense result */
    ogpu::Tri dense[OG_MAX_CALLS]{};
    og_dense_col dense_cols[OG_MAX_CALLS]{};
    ogpu::Scratch bufs; /* the dense record and the plan's scratch: freed by ~og_query after it has synchronised the stream */
    og_stats stats{};
    /* host staging for og_query_next */
    std::vector<uint64_t> h_val[OG_MAX_CALLS];
    std::vector<uint8_t> h_ok[OG_MAX_CALLS];
    std::vector<int64_t> h_tim[OG_MAX_CALLS];
    bool host_ready = false;
    uint32_t next_group = 0, next_row = 0;
    /* record view backing store */
    std::vector<std::vector<uint8_t>> rv_val, rv_bitmap;
    std::vector<std::vector<int64_t>> rv_coltimes;
    std::vector<int64_t> rv_times;
    std::vector<og_colval_view> rv_cols;
    int path_used = 0; /* 0 generic tile path, 1 fused (general kernel), 2 fused Gorilla kernel, per-series cells, 3 fused Gorilla kernel, folded cells, 4 pull-iterator kernel k_fused_multi, 5 column-at-a-time kernel k_fused_cols */
    bool cells_dirty = true; /* per-series cell validity bytes need clearing before the next run */
    /* execution plan + scratch, built by the first og_query_run and reused by later runs */
    bool planned = false;
    uint32_t chunk_series = 0, tile_segs = 0;
    int *d_err = nullptr;
    void *plan = nullptr; /* ogpu::Plan (agg_kernels.cuh types) */
    std::vector<cudaEvent_t> main_ev; /* event pairs around the dominant decode+reduce kernels */
    void *merge_state = nullptr;      /* og_merge_state of the last og_query_allreduce (comm.cu) */
    ~og_query(); /* api.cu */
};
