// common.h -- core types of the auron_b200 engine: data types, device buffers, Arrow-layout
// columns resident in HBM, batches, errors.  Host C++17; included by .cu and .cc files.
//
// Layout in HBM (DESIGN.md "Data layout"): every column is the Arrow columnar layout of the
// reference's RecordBatch (validity bitmap LSB-first, 1 bit/row; fixed-width values; utf8 =
// int32 offsets[n+1] + bytes; bool = bitmap), each buffer a separate stream-ordered allocation
// padded to 16 bytes so 128-bit loads never fault at the tail.
#pragma once
#include <cuda_runtime.h>

#include <cstdint>
#include <cstring>
#include <memory>
#include <stdexcept>
#include <string>
#include <vector>

namespace auron {

struct Error : std::runtime_error {
    using std::runtime_error::runtime_error;
};

[[noreturn]] inline void fail(const std::string& msg) { throw Error(msg); }

#define AURON_CHECK(cond, msg)                                                                  \
    do {                                                                                        \
        if (!(cond)) ::auron::fail(std::string(msg) + " [" #cond "] at " __FILE__ ":" + std::to_string(__LINE__)); \
    } while (0)

#define CUDA_OK(expr)                                                                           \
    do {                                                                                        \
        cudaError_t _e = (expr);                                                                \
        if (_e != cudaSuccess)                                                                  \
            ::auron::fail(std::string("CUDA error: ") + cudaGetErrorString(_e) + " in " #expr " at " __FILE__ ":" + \
                          std::to_string(__LINE__));                                            \
    } while (0)

// ---------------------------------------------------------------------------------------------
// data types (the subset of auron.proto ArrowType :915-951 that reaches the hot path)
// ---------------------------------------------------------------------------------------------
enum TypeId : int32_t {
    T_NULL = 0,
    T_BOOL = 1,
    T_INT8 = 2,
    T_INT16 = 3,
    T_INT32 = 4,
    T_INT64 = 5,
    T_FLOAT32 = 6,
    T_FLOAT64 = 7,
    T_UTF8 = 8,
    T_BINARY = 9,
    T_DATE32 = 10,
    T_DATE64 = 11,
    T_TIMESTAMP = 12,  // int64, unit in DType::unit (0 s, 1 ms, 2 us, 3 ns)
    T_DECIMAL128 = 13,
    T_LIST = 14,       // one level: the element is a flat type (DType::elem); int32 offsets + a child column
};

struct DType {
    TypeId id = T_NULL;
    int32_t precision = 0, scale = 0;  // decimal
    int32_t unit = 2;                  // timestamp unit
    std::string tz;
    // T_LIST: the element's type, and the name and nullability of the child field (kept for the Arrow export)
    std::shared_ptr<const DType> elem;
    std::string elem_name = "item";
    bool elem_nullable = true;
    DType() = default;
    DType(TypeId i) : id(i) {}
    static DType decimal(int p, int s) {
        DType t(T_DECIMAL128);
        t.precision = p;
        t.scale = s;
        return t;
    }
    static DType list(const DType& e, bool nullable = true, const std::string& name = "item") {
        DType t(T_LIST);
        t.elem = std::make_shared<const DType>(e);
        t.elem_nullable = nullable;
        t.elem_name = name;
        return t;
    }
    bool operator==(const DType& o) const {
        if (id != o.id) return false;
        if (id == T_DECIMAL128) return precision == o.precision && scale == o.scale;
        if (id == T_TIMESTAMP) return unit == o.unit;
        if (id == T_LIST) return elem && o.elem && *elem == *o.elem;
        return true;
    }
    bool operator!=(const DType& o) const { return !(*this == o); }
    // byte width of one value; 0 for bool (bitmap), utf8/binary (variable) and null
    int width() const {
        switch (id) {
            case T_INT8: return 1;
            case T_INT16: return 2;
            case T_INT32: case T_FLOAT32: case T_DATE32: return 4;
            case T_INT64: case T_FLOAT64: case T_DATE64: case T_TIMESTAMP: return 8;
            case T_DECIMAL128: return 16;
            default: return 0;
        }
    }
    bool is_varlen() const { return id == T_UTF8 || id == T_BINARY; }
    bool is_integer() const { return id == T_INT8 || id == T_INT16 || id == T_INT32 || id == T_INT64; }
    bool is_intlike() const { return is_integer() || id == T_DATE32 || id == T_DATE64 || id == T_TIMESTAMP; }
    bool is_float() const { return id == T_FLOAT32 || id == T_FLOAT64; }
    std::string str() const;
};

struct Field {
    std::string name;
    DType type;
    bool nullable = true;
};
struct Schema {
    std::vector<Field> fields;
    int index_of(const std::string& name) const {
        for (size_t i = 0; i < fields.size(); i++)
            if (fields[i].name == name) return (int)i;
        return -1;
    }
};

// ---------------------------------------------------------------------------------------------
// execution context: one CUDA stream per task (the reference runs one runtime per Spark task,
// auron/src/rt.rs:75-248); allocations are stream-ordered from the device's default pool.
// ---------------------------------------------------------------------------------------------
struct Ctx {
    int device = 0;
    cudaStream_t stream = nullptr;
    int sm_count = 132;
    int64_t batch_size = 10000;             // auron.batchSize (datafusion-ext-commons/src/lib.rs:72-75)
    int64_t gpu_chunk_rows = 64 << 20;      // device-side accumulation target (SURVEY hard part 2); AURON_GPU_CHUNK_ROWS overrides
    int64_t kernel_launches = 0;            // number of our kernels launched on this ctx
    // stream_priority: 0 = default; < 0 = higher (kernels queued on it get SM slots before those of lower-priority streams)
    explicit Ctx(int dev = 0, int stream_priority = 0);
    ~Ctx();
    Ctx(const Ctx&) = delete;
    void sync();   // cudaStreamSynchronize + recycles the staged-upload arena
    // Small host->device uploads (descriptor tables, page lists) do not go through the copy engine: they are staged
    // in this pinned, device-mapped arena and moved by a tiny kernel on the task stream.  A copy-engine transfer
    // would queue FIFO behind bulk H2D traffic of the scan's prefetch stream.
    uint8_t* stage_host = nullptr;
    size_t stage_cap = 0, stage_off = 0;

    // Optional per-kernel device timing (AURON_PROFILE=1): CUDA events recorded on this stream around named
    // launch sites; bench.py reads the totals through auron_b200_metrics ("__kernels__" pseudo operator).
    struct ProfEntry {
        const char* name;
        cudaEvent_t e0, e1;
    };
    bool profile = false;
    std::vector<ProfEntry> prof;
    struct ProfTotal {
        std::string name;
        double ms = 0;
        int64_t launches = 0;
    };
    std::vector<ProfTotal> prof_summary();   // synchronises; drains the event list
};

struct ProfScope {
    Ctx& ctx;
    bool on;
    cudaEvent_t e0 = nullptr, e1 = nullptr;
    const char* name;
    ProfScope(Ctx& c, const char* n) : ctx(c), on(c.profile), name(n) {
        if (on) {
            cudaEventCreate(&e0);
            cudaEventCreate(&e1);
            cudaEventRecord(e0, ctx.stream);
        }
    }
    ~ProfScope() {
        if (on) {
            cudaEventRecord(e1, ctx.stream);
            ctx.prof.push_back({name, e0, e1});
        }
    }
};

struct DevMem {
    void* ptr = nullptr;
    size_t bytes = 0;
    cudaStream_t stream = nullptr;
    ~DevMem();
};
using Buf = std::shared_ptr<DevMem>;

Buf dalloc(Ctx& ctx, size_t bytes);                  // uninitialised, padded (+64 B)
Buf dalloc_zero(Ctx& ctx, size_t bytes);
Buf dalloc_fill(Ctx& ctx, size_t bytes, int byte);   // memset
Buf to_device(Ctx& ctx, const void* host, size_t bytes);
void upload_small(Ctx& ctx, void* dev, const void* host, size_t bytes);   // 16-byte aligned `dev`, <= 4 MB: staged + kernel, else copy engine
void to_host(Ctx& ctx, void* host, const void* dev, size_t bytes);   // synchronises
template <typename T>
inline T* P(const Buf& b) { return b ? static_cast<T*>(b->ptr) : nullptr; }

// ---------------------------------------------------------------------------------------------
// column / batch
// ---------------------------------------------------------------------------------------------
struct Column {
    DType type;
    int64_t len = 0;
    // null_count: 0 = no nulls (validity may be absent); -1 = unknown, validity present
    int64_t null_count = 0;
    Buf validity;  // bitmap, bit i of byte i/8 (LSB first); nullptr => all valid
    Buf data;      // values; bool => bitmap; utf8/binary => bytes
    Buf offsets;   // int32[len+1] for utf8/binary and list
    int64_t data_bytes = 0;  // utf8/binary: number of payload bytes (== offsets[len])
    // optional bounds of the non-null values of an integer column (a superset is fine): set by the Parquet scan from the
    // column-chunk statistics, used by the aggregate's direct-address path instead of a min/max pass over the keys
    bool has_range = false;
    int64_t range_min = 0, range_max = 0;
    // list: the elements of every row, row i owning child rows [offsets[i], offsets[i+1]) (offsets[0] == 0)
    std::shared_ptr<Column> child;

    const uint8_t* vbits() const { return validity ? static_cast<const uint8_t*>(validity->ptr) : nullptr; }
    bool may_have_nulls() const { return validity != nullptr; }
};
using ColumnPtr = std::shared_ptr<Column>;

struct Batch {
    std::vector<ColumnPtr> cols;
    int64_t num_rows = 0;
};
using BatchPtr = std::shared_ptr<Batch>;

inline int64_t bitmap_bytes(int64_t n) { return (n + 7) / 8; }
// bitmaps are allocated in whole 32-bit words (kernels write them a word at a time)
inline int64_t bitmap_alloc_bytes(int64_t n) { return ((n + 31) / 32) * 4; }

ColumnPtr make_column(Ctx& ctx, const DType& t, int64_t len, bool with_validity);   // fixed-width / bool only
ColumnPtr make_null_column(Ctx& ctx, const DType& t, int64_t len);

}  // namespace auron
