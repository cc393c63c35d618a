/* Host-side mirror of the reference's cursor seam, written above the C ABI (include/ogpu.h).
 *
 * The reference is Go and this image has no Go toolchain, so the shim a maintainer would write in Go (INTEGRATION.md shows
 * it) is mirrored here in C++ with the reference's names, argument meaning and error behaviour:
 *
 *   comm.KeyCursor            engine/comm/cursor.go:46-56      -> ogpu::KeyCursor
 *   comm.CallOption           engine/comm/cursor.go (CallOption{Call, Ref}) -> ogpu::CallOption
 *   record.Record / ColVal    lib/record/record.go:57-61, column.go:30-37   -> ogpu::Record / ogpu::ColVal (borrowed views)
 *   record.Field / Schemas    lib/record/record.go (Field{Type,Name})       -> ogpu::Field / ogpu::Schemas
 *   query.ProcessorOptions    lib/util/lifted/influx/query/select.go (Interval, StartTime, EndTime, Ascending, ChunkSize)
 *   aggregateCursor           engine/aggregate_cursor.go:39-412  \
 *   AggTagSetCursor           engine/agg_tagset_cursor.go:563-1160 } -> ogpu::GpuAggCursor (one object replaces the stack
 *   fileLoopCursor/tsmMerge…  engine/file_cursor.go, tsm_merge_cursor.go /   seriesCursor..AggTagSetCursor of SURVEY §3.1)
 *
 * Contract kept from the reference:
 *   - Next()/NextAggData() return a *borrowed* Record; it stays valid until the next call on the same cursor (the reference's
 *     CircularRecordPool ring, engine/iterators.go:61-70).  End of stream is (nullptr, nullptr, no error) — cursor.go:46-56.
 *   - SetOps before SinkPlan; SinkPlan derives the output schema (call columns in ops order, then "time"; tags removed) the
 *     way aggregateCursor.SinkPlan does (aggregate_cursor.go:208-242).
 *   - Errors are values (Go `error`): every call that can fail returns an Error with code = the C-ABI status and the
 *     library's message.  A cursor is confined to one thread at a time (SURVEY §8b Threading).
 *   - There is no CPU path: if libogpu.so cannot bind an H100 every call fails with OG_E_CUDA.
 */
#pragma once
#include <cstdint>
#include <cstring>
#include <memory>
#include <string>
#include <vector>

#include "../../include/ogpu.h"

namespace ogpu {

/* influx.Field_Type_* (lib/util/lifted/vm/protoparser/influx) — same numeric values as OG_TYPE_* */
enum FieldType : int { Field_Type_Int = 1, Field_Type_Float = 3, Field_Type_String = 4, Field_Type_Boolean = 5 };

struct Field { int Type; std::string Name; };
using Schemas = std::vector<Field>;
inline constexpr const char *TimeField = "time"; /* record.TimeField */

struct Error {
    int code = OG_OK;
    std::string msg;
    explicit operator bool() const { return code != OG_OK; }
    const char *Error_() const { return msg.c_str(); }
};

/* record.ColVal (column.go:30-37).  Views into library-owned host memory. */
struct ColVal {
    const uint8_t *Val = nullptr; size_t ValBytes = 0;
    const uint8_t *Bitmap = nullptr;
    int BitMapOffset = 0, Len = 0, NilCount = 0;
    bool IsNil(int i) const { int b = BitMapOffset + i; return !((Bitmap[b >> 3] >> (b & 7)) & 1); } /* column.go:489-498 */
    const double *FloatValues() const { return reinterpret_cast<const double *>(Val); }
    const int64_t *IntegerValues() const { return reinterpret_cast<const int64_t *>(Val); }
    const uint8_t *BooleanValues() const { return Val; }
};

struct RecMeta { std::vector<const int64_t *> Times; /* per call column, nullptr when absent (record_meta.go:18-26) */ };

struct Record {
    Schemas Schema;              /* field columns then time — time is always last (record.go:57-61) */
    std::vector<ColVal> ColVals; /* same order; ColVals.back() is the time column */
    RecMeta Meta;
    int RowNums() const { return ColVals.empty() ? 0 : ColVals.back().Len; }
    const int64_t *Times() const { return ColVals.back().IntegerValues(); }
};

/* comm.SeriesInfoIntf — only the sid is known to the GPU library; keys/tags stay with the Go index. */
struct SeriesInfo { uint64_t sid = 0; uint32_t group = 0; uint64_t GetSid() const { return sid; } };
struct FileInfo { int64_t MinTime = 0, MaxTime = 0; SeriesInfo Info; };

/* comm.CallOption: Call.Name in {"count","sum","min","max","first","last"}; Ref = field name. */
struct CallOption { std::string Call; std::string Ref; };

/* One leaf of the WHERE condition in RPN, the shape binaryfilterfunc.ConditionImpl compiles to (functions.go:457-837). */
struct CondItem { int kind; std::string field; int op; bool is_float; double f; int64_t i; };

/* The subset of query.ProcessorOptions + hybridqp.QueryNode the cursor reads (select.go:579-640, aggregate_cursor.go:208). */
struct QueryPlan {
    int64_t Interval = 0, Offset = 0;      /* opt.Interval.Duration / .Offset, ns */
    int64_t StartTime = INT64_MIN, EndTime = INT64_MAX;
    bool Ascending = true;
    int ChunkSize = 1000;                  /* opt.ChunkSize → ChunkSizeNum slicing of interval records */
    enum Dims { GroupAll, GroupBySeries, GroupByTagSet } GroupBy = GroupAll;
    std::vector<uint32_t> SeriesGroup;     /* GroupByTagSet: series index → tagset ordinal (from the index scan) */
    uint32_t NumGroups = 1;
    std::vector<CondItem> Condition;       /* RPN */
    bool StrictOrder = false;
};

class KeyCursor { /* engine/comm/cursor.go:46-56 */
public:
    virtual ~KeyCursor() = default;
    virtual void SetOps(const std::vector<CallOption> &ops) = 0;
    virtual Error SinkPlan(const QueryPlan &plan) = 0;
    virtual Error Next(const Record **rec, const SeriesInfo **info) = 0;
    virtual const char *Name() const = 0;
    virtual Error Close() = 0;
    virtual const Schemas &GetSchema() const = 0;
    virtual void StartSpan(void *span) = 0;
    virtual void EndSpan() = 0;
    virtual Error NextAggData(const Record **rec, const FileInfo **info) = 0;
};

/* A shard resident in HBM (immutable.TSSPFile set of one shard; tssp_reader.go).  Ref-counted like tsspFile.Ref/Unref. */
class GpuShard {
public:
    static Error Open(const og_shard_desc &desc, std::shared_ptr<GpuShard> *out);
    static Error Synth(const og_synth_desc &desc, std::shared_ptr<GpuShard> *out);
    ~GpuShard();
    og_shard *handle() const { return s_; }
    const Schemas &schema() const { return schema_; }
    void set_schema(Schemas s) { schema_ = std::move(s); }
private:
    og_shard *s_ = nullptr;
    Schemas schema_;
};

class GpuAggCursor final : public KeyCursor {
public:
    explicit GpuAggCursor(std::shared_ptr<GpuShard> shard);
    ~GpuAggCursor() override;
    void SetOps(const std::vector<CallOption> &ops) override;
    Error SinkPlan(const QueryPlan &plan) override;
    Error Next(const Record **rec, const SeriesInfo **info) override;
    const char *Name() const override { return "gpu_agg_cursor"; }
    Error Close() override;
    const Schemas &GetSchema() const override { return out_schema_; }
    void StartSpan(void *) override { span_ = true; }
    void EndSpan() override;
    Error NextAggData(const Record **rec, const FileInfo **info) override;
    const og_stats &Stats() const { return stats_; }

private:
    Error run_once();
    std::shared_ptr<GpuShard> shard_;
    std::vector<CallOption> ops_;
    Schemas out_schema_;
    og_query *q_ = nullptr;
    bool ran_ = false, closed_ = false, span_ = false;
    Record rec_[2]; int ring_ = 0; /* aggregate cursors own a ring of 2 (iterators.go:61-70) */
    SeriesInfo info_; FileInfo finfo_;
    og_stats stats_{};
};

} // namespace ogpu
