// engine.h -- host runtime: operators (the mirror of DataFusion's ExecutionPlan / RecordBatchStream
// surface used by datafusion-ext-plans), the task runtime (auron/src/rt.rs NativeExecutionRuntime) and
// the planner (auron-planner/src/planner.rs PhysicalPlanner::create_plan).
#pragma once
#include <chrono>
#include <functional>
#include <map>
#include <memory>
#include <string>

#include "arrow_bridge.h"
#include "common.h"
#include "expr.h"
#include "kernels.h"

struct auron_callbacks;   // include/auron_b200.h

namespace auron {

struct Task;

struct MetricSet {
    std::vector<std::pair<std::string, int64_t>> values;
    void add(const std::string& name, int64_t v) {
        for (auto& kv : values)
            if (kv.first == name) {
                kv.second += v;
                return;
            }
        values.emplace_back(name, v);
    }
};

// inclusive wall-clock timer feeding a metric (the reference's elapsed_compute / *_time metrics, execution_context.rs:136-144)
struct OpTimer {
    MetricSet& m;
    const char* name;
    std::chrono::steady_clock::time_point t0;
    OpTimer(MetricSet& ms, const char* n) : m(ms), name(n), t0(std::chrono::steady_clock::now()) {}
    ~OpTimer() { m.add(name, std::chrono::duration_cast<std::chrono::nanoseconds>(std::chrono::steady_clock::now() - t0).count()); }
};

// A batch plus an optional pending row selection (a filter whose gather has not been materialised)
struct SelBatch {
    BatchPtr batch;
    Buf sel;          // int32 row indices into batch (materialised selection), or nullptr
    Buf mask;         // pending selection as a bit mask over the batch rows (bits past num_rows are zero), or nullptr;
                      // consumers that can skip rows themselves (hash aggregate) use it directly, others call ensure_sel()
    int64_t n = 0;    // selected row count (== batch rows when neither sel nor mask is set)
};
struct Task;
const int32_t* ensure_sel(Task& t, SelBatch& s);   // materialise mask -> indices if needed; nullptr = all rows

// ExecutionPlan + RecordBatchStream in one object: execute() == first next()
struct Operator {
    std::string name;
    Schema out_schema;
    std::vector<std::unique_ptr<Operator>> children;
    MetricSet metrics;
    virtual ~Operator() = default;
    virtual BatchPtr next(Task& t) = 0;          // nullptr at end of stream
    // operator-specific attributes as JSON members (`"k":v,...`, no braces) for auron_b200_explain; "" = none
    virtual std::string describe() const { return ""; }
    virtual SelBatch next_sel(Task& t) {         // default: no pending selection
        SelBatch s;
        s.batch = next(t);
        s.n = s.batch ? s.batch->num_rows : 0;
        return s;
    }
};
using OperatorPtr = std::unique_ptr<Operator>;

struct Task {
    Ctx ctx;
    const auron_callbacks* cb = nullptr;
    uint32_t stage_id = 0, partition_id = 0;
    uint64_t task_id = 0;
    OperatorPtr root;
    std::string error;
    bool cancelled = false;
    bool is_running();
    // configuration entry: the host's value (get_conf callback), else the environment variable `env`, else `dflt`
    std::string conf(const char* key, const char* env, const char* dflt) const;
    explicit Task(int device) : ctx(device) {}
};

// process-wide registry of device-resident inputs (bench "value" leg; also build-side caches keyed by
// broadcast id like broadcast_join_exec.rs:579-625)
void put_device_resource(const std::string& id, std::vector<BatchPtr> batches, const Schema& schema);
bool get_device_resource(const std::string& id, std::vector<BatchPtr>* batches, Schema* schema);
void drop_device_resource(const std::string& id);

// Parquet files whose bytes are resident in HBM (scan decodes page payloads in place)
void put_device_file(const std::string& path, const uint8_t* bytes, size_t len, int device);
void drop_device_file(const std::string& path);
void put_host_file(const std::string& path, const uint8_t* bytes, size_t len);
void drop_host_file(const std::string& path);

// expression tree as text, e.g. `Gt(col(a), lit(int32:5))` (plan explain / error messages)
std::string expr_to_string(const Expr& e);
std::string json_quote(const std::string& s);
// planner: TaskDefinition bytes -> Task (operator tree)
std::unique_ptr<Task> create_task(const uint8_t* task_def, size_t len, const auron_callbacks* cb, int device);

Literal decode_scalar_ipc(const uint8_t* bytes, size_t n);
// a flat Arrow array held on the host (the child of a one-row List ScalarValue: range-partition bounds)
struct HostArray {
    DType type;
    int64_t len = 0;
    std::vector<uint8_t> validity;   // empty = no nulls
    std::vector<uint8_t> data;       // values (bool: bitmap; utf8/binary: bytes)
    std::vector<int32_t> offsets;    // utf8/binary
    // the list row itself (list literals): NULL, and the name / nullability of its element field
    bool list_is_null = false;
    std::string elem_name = "item";
    bool elem_nullable = true;
};
bool is_list_scalar_ipc(const uint8_t* bytes, size_t n);   // a ScalarValue whose type is List
HostArray decode_list_scalar_ipc(const uint8_t* bytes, size_t n);
ColumnPtr host_array_to_device(Ctx& ctx, const HostArray& a);

// operators implemented outside engine.cc
OperatorPtr make_parquet_scan(Task& t, const uint8_t* node, size_t n);
OperatorPtr make_shuffle_writer(Task& t, OperatorPtr input, const uint8_t* node, size_t n);
OperatorPtr make_ipc_reader(Task& t, const Schema& schema, const std::string& resource_id);
OperatorPtr make_ipc_writer(Task& t, OperatorPtr input, const std::string& consumer_resource_id);

// expression decode (shared by planner + scan pruning)
ExprPtr decode_expr(const uint8_t* b, size_t n);
Schema decode_schema(const uint8_t* b, size_t n);
DType decode_arrow_type(const uint8_t* b, size_t n);

}  // namespace auron
