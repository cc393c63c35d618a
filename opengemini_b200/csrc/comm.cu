/*
 * comm.cu — the cross-shard merge behind the C ABI: og_comm_* / og_query_allreduce.
 *
 * Replaces the reference's partial-aggregate exchange between store nodes and the sql node
 * (engine/executor/rpc_transform.go:40-282 + agg_transform.go:248-304: every shard's dense interval record is merged
 * column by column with the Update* functions of lib/record/reccord_functions.go).  Here the shards live one per GPU and the
 * merge is
 *     count / sum columns (and their validity)   one ncclAllReduce(sum) over a packed f64 buffer + one over a packed i64 buffer
 *     min / max / first / last columns           one ncclAllGather of the packed (value, time, valid) cells of all ranks, folded
 *                                                 in rank order by k_gather_fold with the reference's tie-break rules
 *                                                 (reccord_functions.go:482-494), so every rank ends with the same record
 * The whole step (pack kernel, <= 3 collectives, unpack/fold kernel) is captured into a CUDA graph on first use and replayed.
 * NCCL is loaded at run time (dlopen libnccl.so.2): a single-GPU host needs no NCCL at all.
 */
#include <dlfcn.h>

#include <cstdio>
#include <cstdlib>
#include <cstring>

#include "agg_ops.cuh"
#include "internal.h"

namespace {

/* ---- the part of nccl.h this file needs (NCCL 2.x ABI) ---- */
typedef struct ncclComm *ncclComm_t;
typedef struct { char internal[128]; } ncclUniqueId;
typedef enum { ncclSuccess = 0 } ncclResult_t;
typedef enum { ncclInt8 = 0, ncclChar = 0, ncclUint8 = 1, ncclInt32 = 2, ncclUint32 = 3, ncclInt64 = 4, ncclUint64 = 5, ncclFloat16 = 6, ncclFloat32 = 7, ncclFloat64 = 8 } ncclDataType_t;
typedef enum { ncclSum = 0, ncclProd = 1, ncclMax = 2, ncclMin = 3 } ncclRedOp_t;
struct NcclApi {
    void *h = nullptr;
    ncclResult_t (*GetUniqueId)(ncclUniqueId *) = nullptr;
    ncclResult_t (*CommInitRank)(ncclComm_t *, int, ncclUniqueId, int) = nullptr;
    ncclResult_t (*CommDestroy)(ncclComm_t) = nullptr;
    ncclResult_t (*AllReduce)(const void *, void *, size_t, ncclDataType_t, ncclRedOp_t, ncclComm_t, cudaStream_t) = nullptr;
    ncclResult_t (*AllGather)(const void *, void *, size_t, ncclDataType_t, ncclComm_t, cudaStream_t) = nullptr;
    ncclResult_t (*GroupStart)() = nullptr;
    ncclResult_t (*GroupEnd)() = nullptr;
    const char *(*GetErrorString)(ncclResult_t) = nullptr;
    ncclResult_t (*GetVersion)(int *) = nullptr;
};
NcclApi g_nccl;
std::mutex g_nccl_mu;

int load_nccl() {
    std::lock_guard<std::mutex> lock(g_nccl_mu);
    if (g_nccl.h) return OG_OK;
    const char *cands[] = {getenv("OGPU_NCCL_LIB"), "libnccl.so.2", "libnccl.so"};
    void *h = nullptr;
    for (const char *c : cands) { if (c && *c && (h = dlopen(c, RTLD_NOW | RTLD_GLOBAL))) break; }
    if (!h) { ogpu::set_error("NCCL not found (dlopen libnccl.so.2: %s); set OGPU_NCCL_LIB", dlerror()); return OG_E_UNSUPPORTED; }
#define SYM(name) do { *(void **)&g_nccl.name = dlsym(h, "nccl" #name); if (!g_nccl.name) { ogpu::set_error("libnccl lacks nccl" #name); dlclose(h); return OG_E_UNSUPPORTED; } } while (0)
    SYM(GetUniqueId); SYM(CommInitRank); SYM(CommDestroy); SYM(AllReduce); SYM(AllGather); SYM(GroupStart); SYM(GroupEnd); SYM(GetErrorString); SYM(GetVersion);
#undef SYM
    g_nccl.h = h;
    return OG_OK;
}
#define NC(call) do { ncclResult_t r__ = (call); if (r__ != ncclSuccess) { ogpu::set_error("NCCL error %d (%s) at %s:%d: %s", (int)r__, g_nccl.GetErrorString(r__), __FILE__, __LINE__, #call); return OG_E_CUDA; } } while (0)

} // namespace

struct og_comm {
    ncclComm_t comm = nullptr;
    int rank = 0, world = 1, device = 0;
};

namespace ogpu {

struct DenseP { Tri dense[OG_MAX_CALLS]; }; /* the query's dense interval record (device arrays) */

/* what one merge moves, per call column: where it sits in the packed buffers */
struct MergeCol { int32_t func, type, kind; /* 0 sum f64, 1 sum i64 (count / integer sum), 2 gathered selector */ uint32_t slot; int32_t has_time; };
struct MergeP {
    uint32_t n_cols, n_f64, n_i64, n_sel, world;
    uint64_t cells;
    MergeCol cols[OG_MAX_CALLS];
    double *f64;   /* [n_f64][cells] values of float sums (invalid cells = 0) */
    int64_t *i64;  /* [n_i64 + n_f64 + n_i64][cells]: integer sums/counts, then one validity plane (0/1) per summed column */
    uint64_t *sel_send, *sel_recv; /* selectors: per column {value u64, time i64, valid u64} planes: [n_sel][3][cells]; recv = [world] of those */
};

__global__ void k_merge_pack(QueryP q, DenseP g, MergeP m) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= m.cells) return;
    uint32_t vplane = m.n_i64;
    for (uint32_t c = 0; c < m.n_cols; c++) {
        const MergeCol &mc = m.cols[c];
        const uint32_t ok = g.dense[c].ok[i];
        const uint64_t v = ok ? g.dense[c].val[i] : 0;
        if (mc.kind == 0) { m.f64[(uint64_t)mc.slot * m.cells + i] = ok ? u2d(v) : 0.0; m.i64[(uint64_t)(vplane++) * m.cells + i] = ok; }
        else if (mc.kind == 1) { m.i64[(uint64_t)mc.slot * m.cells + i] = (int64_t)v; m.i64[(uint64_t)(vplane++) * m.cells + i] = ok; }
        else {
            uint64_t *p = m.sel_send + (uint64_t)mc.slot * 3 * m.cells;
            p[i] = v; p[m.cells + i] = (uint64_t)(g.dense[c].tim ? g.dense[c].tim[i] : 0); p[2 * m.cells + i] = ok;
        }
    }
}

/* after the collectives: sums/counts are final; selectors fold the gathered cells of all ranks in rank order, starting from an
 * empty interval-record cell, with the tagset update rules — identical on every rank */
__global__ void k_merge_unpack(QueryP q, DenseP g, MergeP m) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= m.cells) return;
    uint32_t vplane = m.n_i64;
    const uint32_t b = (uint32_t)(i % q.n_buckets);
    for (uint32_t c = 0; c < m.n_cols; c++) {
        const MergeCol &mc = m.cols[c];
        if (mc.kind == 0) { const int64_t ok = m.i64[(uint64_t)(vplane++) * m.cells + i]; g.dense[c].val[i] = ok ? d2u(m.f64[(uint64_t)mc.slot * m.cells + i]) : 0; g.dense[c].ok[i] = ok != 0; }
        else if (mc.kind == 1) { const int64_t ok = m.i64[(uint64_t)(vplane++) * m.cells + i]; g.dense[c].val[i] = ok ? (uint64_t)m.i64[(uint64_t)mc.slot * m.cells + i] : 0; g.dense[c].ok[i] = ok != 0; }
        else {
            Part a; a.v = 0; a.ok = 0; a.t = (mc.has_time && !q.multi) ? q.start + (int64_t)b * q.interval : 0;
            const uint64_t stride = (uint64_t)m.n_sel * 3 * m.cells;
            for (uint32_t r = 0; r < m.world; r++) {
                const uint64_t *p = m.sel_recv + r * stride + (uint64_t)mc.slot * 3 * m.cells;
                Part x; x.v = p[i]; x.t = (int64_t)p[m.cells + i]; x.ok = (uint32_t)p[2 * m.cells + i];
                group_update(mc.func, mc.type, q.multi != 0, a, x);
            }
            g.dense[c].val[i] = a.v; g.dense[c].ok[i] = (uint8_t)a.ok;
            if (g.dense[c].tim) g.dense[c].tim[i] = a.t;
        }
    }
}

} // namespace ogpu

using namespace ogpu;

struct og_merge_state { /* per (query, communicator): buffers + the captured graph */
    og_comm *comm = nullptr;
    MergeP mp{};
    cudaGraphExec_t graph = nullptr;
    bool geometry_checked = false;
    Scratch bufs; /* the packed buffers of mp */
    ~og_merge_state() { if (graph) cudaGraphExecDestroy(graph); }
};

extern "C" {

OG_API int og_comm_unique_id(uint8_t id[128]) {
    if (!id) return OG_E_INVAL;
    int rc = load_nccl(); if (rc) return rc;
    ncclUniqueId u;
    NC(g_nccl.GetUniqueId(&u));
    memcpy(id, u.internal, 128);
    return OG_OK;
}

OG_API int og_comm_init_rank(const uint8_t id[128], int rank, int world, og_comm **out) {
    if (!id || !out || world < 1 || rank < 0 || rank >= world) { set_error("bad communicator arguments"); return OG_E_INVAL; }
    *out = nullptr;
    int rc = load_nccl(); if (rc) return rc;
    if ((rc = ensure_device())) return rc;
    og_comm *c = new og_comm;
    c->rank = rank; c->world = world;
    cudaGetDevice(&c->device);
    ncclUniqueId u; memcpy(u.internal, id, 128);
    ncclResult_t r = g_nccl.CommInitRank(&c->comm, world, u, rank);
    if (r != ncclSuccess) { set_error("ncclCommInitRank failed: %s", g_nccl.GetErrorString(r)); delete c; return OG_E_CUDA; }
    *out = c;
    return OG_OK;
}

OG_API void og_comm_destroy(og_comm *c) {
    if (!c) return;
    if (c->comm && g_nccl.CommDestroy) g_nccl.CommDestroy(c->comm);
    delete c;
}

OG_API int og_comm_info(const og_comm *c, int *rank, int *world, int *nccl_version) {
    if (!c) return OG_E_INVAL;
    if (rank) *rank = c->rank;
    if (world) *world = c->world;
    if (nccl_version && g_nccl.GetVersion) g_nccl.GetVersion(nccl_version);
    return OG_OK;
}

/* sum of `n` doubles over all ranks, in place on the host (timing / row-count plumbing for callers without another channel) */
OG_API int og_comm_allreduce_f64(og_comm *c, double *vals, int n, int op_max) {
    if (!c || !vals || n <= 0 || n > 64) return OG_E_INVAL;
    CU(cudaSetDevice(c->device));
    Scratch tmp;
    double *d; int rc = tmp.get(&d, (size_t)n); if (rc) return rc;
    CU(cudaMemcpy(d, vals, (size_t)n * 8, cudaMemcpyHostToDevice));
    ncclResult_t r = g_nccl.AllReduce(d, d, (size_t)n, ncclFloat64, op_max ? ncclMax : ncclSum, c->comm, nullptr);
    cudaError_t e = cudaMemcpy(vals, d, (size_t)n * 8, cudaMemcpyDeviceToHost);
    if (r != ncclSuccess) { set_error("ncclAllReduce failed: %s", g_nccl.GetErrorString(r)); return OG_E_CUDA; }
    if (e != cudaSuccess) return cuda_fail(e, "allreduce copy", __FILE__, __LINE__);
    return OG_OK;
}

void og_query_free_merge_state(void *p) { delete (og_merge_state *)p; }

static int enqueue_merge(og_query *q, og_merge_state *ms, cudaStream_t st) {
    const MergeP &m = ms->mp;
    DenseP g; memset(&g, 0, sizeof g);
    for (uint32_t c = 0; c < q->qp.n_calls; c++) g.dense[c] = q->dense[c];
    const unsigned blocks = (unsigned)((m.cells + 255) / 256);
    k_merge_pack<<<blocks, 256, 0, st>>>(q->qp, g, m);
    NC(g_nccl.GroupStart());
    if (m.n_f64) NC(g_nccl.AllReduce(m.f64, m.f64, (size_t)m.n_f64 * m.cells, ncclFloat64, ncclSum, ms->comm->comm, st));
    if (m.n_i64 + m.n_f64) NC(g_nccl.AllReduce(m.i64, m.i64, (size_t)(2 * m.n_i64 + m.n_f64) * m.cells, ncclInt64, ncclSum, ms->comm->comm, st));
    if (m.n_sel) NC(g_nccl.AllGather(m.sel_send, m.sel_recv, (size_t)m.n_sel * 3 * m.cells, ncclUint64, ms->comm->comm, st));
    NC(g_nccl.GroupEnd());
    k_merge_unpack<<<blocks, 256, 0, st>>>(q->qp, g, m);
    CU(cudaGetLastError());
    return OG_OK;
}

/* merge this query's dense interval record with the same query's record on every other rank of `c`, in place */
OG_API int og_query_allreduce(og_query *q, og_comm *c) {
    if (!q || !c) return OG_E_INVAL;
    if (!q->ran) { set_error("og_query_allreduce before og_query_run"); return OG_E_STATE; }
    CU(cudaSetDevice(q->sh->device));
    const QueryP &p = q->qp;
    cudaStream_t st = q->stream;
    og_merge_state *ms = (og_merge_state *)q->merge_state;
    if (ms && ms->comm != c) { delete ms; ms = nullptr; q->merge_state = nullptr; }
    if (!ms) { /* the query keeps it once its buffers are allocated */
        std::unique_ptr<og_merge_state> nm(new og_merge_state); nm->comm = c;
        MergeP &m = nm->mp;
        m.n_cols = p.n_calls; m.world = (uint32_t)c->world; m.cells = (uint64_t)q->n_groups * p.n_buckets;
        for (uint32_t k = 0; k < p.n_calls; k++) {
            MergeCol &mc = m.cols[k];
            mc.func = p.calls[k].func; mc.type = p.calls[k].func == OG_AGG_COUNT ? OG_TYPE_INT : p.calls[k].type; mc.has_time = q->dense[k].tim != nullptr;
            if (mc.func == OG_AGG_SUM && mc.type == OG_TYPE_FLOAT) { mc.kind = 0; mc.slot = m.n_f64++; }
            else if (mc.func == OG_AGG_SUM || mc.func == OG_AGG_COUNT) { mc.kind = 1; mc.slot = m.n_i64++; }
            else { mc.kind = 2; mc.slot = m.n_sel++; }
        }
        int rc;
        if (m.n_f64 && (rc = nm->bufs.get(&m.f64, (size_t)m.n_f64 * m.cells))) return rc;
        if (m.n_f64 + m.n_i64 && (rc = nm->bufs.get(&m.i64, (size_t)(2 * m.n_i64 + m.n_f64) * m.cells))) return rc;
        if (m.n_sel && ((rc = nm->bufs.get(&m.sel_send, (size_t)m.n_sel * 3 * m.cells)) || (rc = nm->bufs.get(&m.sel_recv, (size_t)m.world * m.n_sel * 3 * m.cells)))) return rc;
        q->merge_state = ms = nm.release();
    }
    if (!ms->geometry_checked) { /* every rank must hold the same grid and the same calls: compare a fingerprint through the communicator */
        double fp[8] = {(double)p.n_buckets, (double)q->n_groups, (double)p.n_calls, (double)(p.start >> 20), (double)(p.start & 0xfffff), (double)(p.interval >> 20), (double)(p.interval & 0xfffff), 0.0};
        for (uint32_t k = 0; k < p.n_calls; k++) fp[7] = fp[7] * 7.0 + p.calls[k].func + 0.5 * p.calls[k].type;
        double lo[8], hi[8];
        memcpy(lo, fp, sizeof fp); memcpy(hi, fp, sizeof fp);
        for (int k = 0; k < 8; k++) lo[k] = -lo[k];
        int rc = og_comm_allreduce_f64(c, lo, 8, 1); if (rc) return rc;
        rc = og_comm_allreduce_f64(c, hi, 8, 1); if (rc) return rc;
        for (int k = 0; k < 8; k++) if (-lo[k] != hi[k]) {
            set_error("ranks disagree on the dense grid or the calls (field %d: min %.0f max %.0f): create every rank's query with OG_Q_QUERY_GRID and the same descriptor", k, -lo[k], hi[k]);
            return OG_E_INVAL;
        }
        ms->geometry_checked = true;
    }
    cudaEvent_t e0 = q->ev0, e1 = q->ev1;
    CU(cudaEventRecord(e0, st));
    if (!ms->graph && !getenv("OGPU_NO_MERGE_GRAPH")) { /* capture once: pack, collectives, unpack */
        cudaGraph_t graph = nullptr;
        if (cudaStreamBeginCapture(st, cudaStreamCaptureModeThreadLocal) == cudaSuccess) {
            int rc = enqueue_merge(q, ms, st);
            cudaError_t ce = cudaStreamEndCapture(st, &graph);
            if (rc == OG_OK && ce == cudaSuccess && graph && cudaGraphInstantiate(&ms->graph, graph, 0) == cudaSuccess) { /* captured */ }
            else { cudaGetLastError(); ms->graph = nullptr; }
            if (graph) cudaGraphDestroy(graph);
        } else cudaGetLastError();
    }
    if (ms->graph) CU(cudaGraphLaunch(ms->graph, st));
    else { int rc = enqueue_merge(q, ms, st); if (rc) return rc; }
    CU(cudaEventRecord(e1, st));
    CU(cudaStreamSynchronize(st));
    float ms_f = 0; cudaEventElapsedTime(&ms_f, e0, e1);
    q->stats.merge_ms = ms_f;
    q->host_ready = false;
    return OG_OK;
}

} // extern "C"
