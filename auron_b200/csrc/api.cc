// api.cc -- the extern "C" boundary (include/auron_b200.h).  Never throws across the ABI: every entry
// point converts engine errors to a return code + thread-local message, the way the reference converts
// Rust errors/panics into a Java exception and a false/0 return (auron/src/lib.rs:30-82, rt.rs:205-236).
#include <algorithm>
#include <atomic>
#include <chrono>
#include <cstring>
#include <mutex>
#include <map>

#include "../../include/auron_b200.h"
#include "exchange.h"
#include "operators.h"
#include "mem_manager.h"
#include "tzdb.h"

using namespace auron;

struct auron_task {
    std::unique_ptr<Task> task;
    bool finished = false;
    int64_t compute_ns = 0, export_ns = 0;   // host wall time inside next_batch: operator tree vs D2H export
};

static thread_local std::string g_last_error;
static std::atomic<int64_t> g_launches{0};

#define API_GUARD_BEGIN try {
#define API_GUARD_END(ret)                \
    }                                     \
    catch (const std::exception& e) {     \
        g_last_error = e.what();          \
        return ret;                       \
    }                                     \
    catch (...) {                         \
        g_last_error = "unknown failure"; \
        return ret;                       \
    }

#pragma GCC visibility push(default)
extern "C" {

const char* auron_b200_last_error(void) { return g_last_error.c_str(); }

auron_task* auron_b200_call_native(const uint8_t* task_definition, size_t len, const auron_callbacks* callbacks, int device) {
    API_GUARD_BEGIN
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) fail("auron_b200 requires a CUDA device (no CPU fallback)");
    auto* h = new auron_task;
    try {
        h->task = create_task(task_definition, len, callbacks, device);
    } catch (...) {
        delete h;
        throw;
    }
    return h;
    API_GUARD_END(nullptr)
}

int auron_b200_schema(auron_task* task, struct ArrowSchema* out) {
    API_GUARD_BEGIN
    AURON_CHECK(task && task->task, "null task");
    schema_to_arrow(task->task->root->out_schema, out);
    return 0;
    API_GUARD_END(-1)
}

int auron_b200_next_batch(auron_task* task, struct ArrowArray* out) {
    API_GUARD_BEGIN
    AURON_CHECK(task && task->task, "null task");
    Task& t = *task->task;
    if (task->finished) return 0;
    CUDA_OK(cudaSetDevice(t.ctx.device));
    int64_t before = t.ctx.kernel_launches;
    BatchPtr b;
    auto t0 = std::chrono::steady_clock::now();
    // WrappedSender::send drops empty batches (execution_context.rs:715-738)
    do {
        b = t.root->next(t);
    } while (b && b->num_rows == 0);
    auto t1 = std::chrono::steady_clock::now();
    task->compute_ns += std::chrono::duration_cast<std::chrono::nanoseconds>(t1 - t0).count();
    g_launches += t.ctx.kernel_launches - before;
    if (!b) {
        task->finished = true;
        return 0;
    }
    export_batch(t.ctx, *b, t.root->out_schema, out);
    task->export_ns += std::chrono::duration_cast<std::chrono::nanoseconds>(std::chrono::steady_clock::now() - t1).count();
    return 1;
    API_GUARD_END(-1)
}

void auron_b200_finalize_native(auron_task* task) {
    if (!task) return;
    try {
        if (task->task) {
            task->task->cancelled = true;
            cudaSetDevice(task->task->ctx.device);
            task->task->root.reset();
            task->task.reset();
        }
    } catch (...) {
    }
    delete task;
}

void auron_b200_on_exit(void) {}

static void walk_metrics(Operator& op, int depth, auron_metric_fn fn, void* user) {
    for (auto& kv : op.metrics.values) fn(user, depth, op.name.c_str(), kv.first.c_str(), kv.second);
    for (auto& c : op.children) walk_metrics(*c, depth + 1, fn, user);
}
int auron_b200_metrics(auron_task* task, auron_metric_fn fn, void* user) {
    API_GUARD_BEGIN
    AURON_CHECK(task && task->task && task->task->root, "null task");
    walk_metrics(*task->task->root, 0, fn, user);
    // device-time totals of the named launch sites (AURON_PROFILE=1), reported under a pseudo operator
    for (auto& k : task->task->ctx.prof_summary()) {
        fn(user, -1, "__kernels__", (k.name + ".device_us").c_str(), (int64_t)(k.ms * 1000.0));
        fn(user, -1, "__kernels__", (k.name + ".launches").c_str(), k.launches);
    }
    fn(user, -1, "__kernels__", "total_launches", task->task->ctx.kernel_launches);
    fn(user, -1, "__task__", "compute_ns", task->compute_ns);
    fn(user, -1, "__task__", "export_ns", task->export_ns);
    return 0;
    API_GUARD_END(-1)
}

static void walk_metric_nodes(Operator& op, int depth, int child_index, auron_metric_node_fn enter, auron_metric_fn fn, void* user) {
    enter(user, depth, child_index, op.name.c_str());
    for (auto& kv : op.metrics.values) fn(user, depth, op.name.c_str(), kv.first.c_str(), kv.second);
    int i = 0;
    for (auto& c : op.children) walk_metric_nodes(*c, depth + 1, i++, enter, fn, user);
}
int auron_b200_metrics_walk(auron_task* task, auron_metric_node_fn enter, auron_metric_fn fn, void* user) {
    API_GUARD_BEGIN
    AURON_CHECK(task && task->task && task->task->root && enter && fn, "null task or callback");
    walk_metric_nodes(*task->task->root, 0, 0, enter, fn, user);
    return 0;
    API_GUARD_END(-1)
}

static void explain_op(const Operator& op, std::string& o) {
    o += "{\"op\":" + json_quote(op.name) + ",\"schema\":[";
    for (size_t i = 0; i < op.out_schema.fields.size(); i++)
        o += std::string(i ? "," : "") + "[" + json_quote(op.out_schema.fields[i].name) + "," + json_quote(op.out_schema.fields[i].type.str()) + "]";
    o += "]";
    const std::string attrs = op.describe();
    if (!attrs.empty()) o += "," + attrs;
    o += ",\"children\":[";
    for (size_t i = 0; i < op.children.size(); i++) {
        if (i) o += ",";
        explain_op(*op.children[i], o);
    }
    o += "]}";
}
int64_t auron_b200_explain(const uint8_t* task_definition, size_t len, char* out, int64_t cap) {
    API_GUARD_BEGIN
    std::unique_ptr<Task> t = create_task(task_definition, len, nullptr, -1);   // device -1: decode only, nothing is launched
    std::string o = "{\"stage_id\":" + std::to_string(t->stage_id) + ",\"partition_id\":" + std::to_string(t->partition_id) + ",\"task_id\":" +
                    std::to_string(t->task_id) + ",\"plan\":";
    explain_op(*t->root, o);
    o += "}";
    if (out && cap > 0) {
        const size_t n = std::min<size_t>(o.size(), (size_t)cap - 1);
        memcpy(out, o.data(), n);
        out[n] = 0;
    }
    return (int64_t)o.size();
    API_GUARD_END(-1)
}

int auron_b200_tz_offset(const char* zone, int64_t utc_second, int32_t* offset) {
    API_GUARD_BEGIN
    AURON_CHECK(zone && offset, "null argument");
    static std::mutex mu;
    static std::map<std::string, TzTable> cache;
    std::lock_guard<std::mutex> g(mu);
    auto it = cache.find(zone);
    if (it == cache.end()) {
        TzTable t;
        if (!load_tz_table(zone, &t)) {
            g_last_error = std::string("unknown time zone ") + zone;
            return -1;
        }
        it = cache.emplace(zone, std::move(t)).first;
    }
    *offset = it->second.offset_at(utc_second);
    return 0;
    API_GUARD_END(-1)
}

int auron_b200_digest_hex(int32_t alg, const uint8_t* bytes, int64_t len, char* out) {
    API_GUARD_BEGIN
    AURON_CHECK(out && len >= 0 && (len == 0 || bytes), "null buffer or negative length");
    if (digest_hex_width(alg) < 0) {
        g_last_error = "unknown digest algorithm " + std::to_string(alg);
        return -1;
    }
    return digest_hex_host(alg, bytes, len, out);
    API_GUARD_END(-1)
}

int auron_b200_float_to_text(int32_t bits, uint64_t value, char* out) {
    API_GUARD_BEGIN
    if (!out || (bits != 32 && bits != 64) || (bits == 32 && value >> 32)) {
        g_last_error = "float_to_text: bits must be 32 or 64, the value a bit pattern of that width, out non-null";
        return -1;
    }
    return float_to_text_host(bits, value, out);
    API_GUARD_END(-1)
}

int auron_b200_text_to_float(int32_t bits, const uint8_t* text, int64_t len, uint64_t* value) {
    API_GUARD_BEGIN
    if (!value || (bits != 32 && bits != 64) || len < 0 || len > INT32_MAX || (len > 0 && !text)) {
        g_last_error = "text_to_float: bits must be 32 or 64, len in 0..2^31-1, text and value non-null";
        return -1;
    }
    return text_to_float_host(bits, text, (int32_t)len, value) ? 1 : 0;
    API_GUARD_END(-1)
}

int64_t auron_b200_zstd_decompress(const uint8_t* in, int64_t in_len, uint8_t* out, int64_t out_len) {
    API_GUARD_BEGIN
    if (in_len < 0 || out_len < 0 || (in_len > 0 && !in) || (out_len > 0 && !out)) {
        g_last_error = "zstd_decompress: lengths must be >= 0 and buffers non-null";
        return -1;
    }
    const int64_t r = zstd_decompress_host(in, in_len, out, out_len);
    if (r < 0) g_last_error = "zstd_decompress: malformed ZSTD data, or more than out_len bytes";
    return r;
    API_GUARD_END(-1)
}

// ---- device residency
static std::map<int, std::unique_ptr<Ctx>>& util_ctxs() {
    static std::map<int, std::unique_ptr<Ctx>> m;
    return m;
}
static Ctx& util_ctx(int device) {
    auto& m = util_ctxs();
    auto it = m.find(device);
    if (it == m.end()) it = m.emplace(device, std::make_unique<Ctx>(device)).first;
    CUDA_OK(cudaSetDevice(device));
    return *it->second;
}

int auron_b200_put_device_batch(const char* resource_id, const struct ArrowArray* batch, const struct ArrowSchema* schema, int device) {
    API_GUARD_BEGIN
    Ctx& ctx = util_ctx(device);
    Schema s = schema_from_arrow(schema);
    BatchPtr b = import_batch(ctx, batch, s);
    put_device_resource(resource_id, {b}, s);
    return 0;
    API_GUARD_END(-1)
}
int64_t auron_b200_set_hbm_budget(int device, int64_t bytes) {
    try {
        return MemManager::of(device).set_budget(bytes);
    } catch (...) {
        return -1;
    }
}
void auron_b200_drop_device_resource(const char* resource_id) {
    try {
        drop_device_resource(resource_id);
    } catch (...) {
    }
}
int auron_b200_put_device_file(const char* path, const uint8_t* bytes, size_t len, int device) {
    API_GUARD_BEGIN
    CUDA_OK(cudaSetDevice(device));
    put_device_file(path, bytes, len, device);
    return 0;
    API_GUARD_END(-1)
}
void auron_b200_drop_device_file(const char* path) {
    try {
        drop_device_file(path);
    } catch (...) {
    }
}
int auron_b200_put_host_file(const char* path, const uint8_t* bytes, size_t len) {
    API_GUARD_BEGIN
    AURON_CHECK(path && bytes, "put_host_file: null argument");
    put_host_file(path, bytes, len);
    return 0;
    API_GUARD_END(-1)
}
void auron_b200_drop_host_file(const char* path) {
    try {
        drop_host_file(path);
    } catch (...) {
    }
}

// ---- NCCL exchange plumbing
int auron_b200_nccl_unique_id(uint8_t out_id[128]) {
    API_GUARD_BEGIN
    nccl_get_unique_id(out_id);
    return 0;
    API_GUARD_END(-1)
}
int auron_b200_nccl_init(const uint8_t id[128], int rank, int world, int device) {
    API_GUARD_BEGIN
    nccl_init(id, rank, world, device);
    return 0;
    API_GUARD_END(-1)
}
void auron_b200_nccl_finalize(void) {
    try {
        nccl_finalize();
    } catch (...) {
    }
}

// ---- kernel-level entry points
static int one_column_out(Ctx& ctx, Buf data, int64_t n, const DType& t, const char* name, struct ArrowArray* out, struct ArrowSchema* out_schema) {
    auto col = std::make_shared<Column>();
    col->type = t;
    col->len = n;
    col->data = data;
    Batch b;
    b.num_rows = n;
    b.cols.push_back(col);
    Schema s;
    Field f;
    f.name = name;
    f.type = t;
    s.fields.push_back(f);
    export_batch(ctx, b, s, out);
    schema_to_arrow(s, out_schema);
    return 0;
}

int auron_b200_k_hash(const struct ArrowArray* batch, const struct ArrowSchema* schema, const int32_t* cols, int32_t ncols, int32_t kind, int64_t seed,
                      struct ArrowArray* out, struct ArrowSchema* out_schema, int device) {
    API_GUARD_BEGIN
    Ctx& ctx = util_ctx(device);
    int64_t before = ctx.kernel_launches;
    Schema s = schema_from_arrow(schema);
    BatchPtr b = import_batch(ctx, batch, s);
    std::vector<ColumnPtr> kc;
    for (int i = 0; i < ncols; i++) {
        AURON_CHECK(cols[i] >= 0 && cols[i] < (int)b->cols.size(), "column index out of range");
        kc.push_back(b->cols[cols[i]]);
    }
    Buf h = hash_columns(ctx, kc, b->num_rows, kind, seed);
    int rc = one_column_out(ctx, h, b->num_rows, DType(kind == 0 ? T_INT32 : T_INT64), "hash", out, out_schema);
    g_launches += ctx.kernel_launches - before;
    return rc;
    API_GUARD_END(-1)
}

int auron_b200_k_partition_ids(const struct ArrowArray* batch, const struct ArrowSchema* schema, const int32_t* cols, int32_t ncols,
                               int32_t num_partitions, struct ArrowArray* out, struct ArrowSchema* out_schema, int device) {
    API_GUARD_BEGIN
    Ctx& ctx = util_ctx(device);
    int64_t before = ctx.kernel_launches;
    Schema s = schema_from_arrow(schema);
    BatchPtr b = import_batch(ctx, batch, s);
    std::vector<ColumnPtr> kc;
    for (int i = 0; i < ncols; i++) {
        AURON_CHECK(cols[i] >= 0 && cols[i] < (int)b->cols.size(), "column index out of range");
        kc.push_back(b->cols[cols[i]]);
    }
    Buf h = murmur3_partition_ids(ctx, kc, b->num_rows, num_partitions, 42);
    int rc = one_column_out(ctx, h, b->num_rows, DType(T_INT32), "partition_id", out, out_schema);
    g_launches += ctx.kernel_launches - before;
    return rc;
    API_GUARD_END(-1)
}

int64_t auron_b200_kernel_launches(void) { return g_launches.load(); }

// average ms per launch of a named kernel over a device-resident resource (CUDA events on the launching stream)
double auron_b200_time_kernel(const char* kernel, const char* resource_id, int32_t iters, int32_t arg0, int device) {
    API_GUARD_BEGIN
    Ctx& ctx = util_ctx(device);
    std::vector<BatchPtr> batches;
    Schema s;
    AURON_CHECK(get_device_resource(resource_id, &batches, &s) && !batches.empty(), std::string("unknown device resource ") + resource_id);
    BatchPtr b = batches[0];
    std::string k(kernel);
    cudaEvent_t e0, e1;
    CUDA_OK(cudaEventCreate(&e0));
    CUDA_OK(cudaEventCreate(&e1));
    auto run = [&]() {
        if (k == "partition_ids") {
            murmur3_partition_ids(ctx, {b->cols[0]}, b->num_rows, arg0 > 0 ? arg0 : 200, 42);
        } else if (k == "agg_sum_count") {   // GROUP BY col0, SUM(col1), COUNT(col1)
            std::vector<AccSpec> specs;
            specs.push_back({ACC_SUM_I64, b->cols[1], {}, DType(T_INT64), nullptr});
            specs.push_back({ACC_COUNT, b->cols[1], {}, DType(T_INT64), nullptr});
            hash_aggregate(ctx, {b->cols[0]}, specs, nullptr, b->num_rows);
        } else fail("unknown kernel " + k);
    };
    run();
    ctx.sync();
    int64_t before = ctx.kernel_launches;
    CUDA_OK(cudaEventRecord(e0, ctx.stream));
    for (int i = 0; i < iters; i++) run();
    CUDA_OK(cudaEventRecord(e1, ctx.stream));
    CUDA_OK(cudaEventSynchronize(e1));
    float ms = 0;
    CUDA_OK(cudaEventElapsedTime(&ms, e0, e1));
    cudaEventDestroy(e0);
    cudaEventDestroy(e1);
    g_launches += ctx.kernel_launches - before;
    return (double)ms / std::max(iters, 1);
    API_GUARD_END(-1.0)
}

}  // extern "C"
#pragma GCC visibility pop
