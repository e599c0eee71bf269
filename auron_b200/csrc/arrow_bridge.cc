// arrow_bridge.cc -- Arrow C Data Interface <-> device columns.
#include "arrow_bridge.h"

#include <memory>

#include "host_pool.h"

#include <cstdlib>

namespace auron {

DType dtype_from_format(const char* f) {
    std::string s(f);
    if (s == "n") return DType(T_NULL);
    if (s == "b") return DType(T_BOOL);
    if (s == "c") return DType(T_INT8);
    if (s == "s") return DType(T_INT16);
    if (s == "i") return DType(T_INT32);
    if (s == "l") return DType(T_INT64);
    if (s == "f") return DType(T_FLOAT32);
    if (s == "g") return DType(T_FLOAT64);
    if (s == "u") return DType(T_UTF8);
    if (s == "z") return DType(T_BINARY);
    if (s == "tdD") return DType(T_DATE32);
    if (s == "tdm") return DType(T_DATE64);
    if (s.rfind("ts", 0) == 0 && s.size() >= 4) {
        DType t(T_TIMESTAMP);
        t.unit = s[2] == 's' ? 0 : s[2] == 'm' ? 1 : s[2] == 'u' ? 2 : 3;
        t.tz = s.substr(4);
        return t;
    }
    if (s.rfind("d:", 0) == 0) {
        int p = 0, sc = 0, bits = 128;
        int n = sscanf(s.c_str(), "d:%d,%d,%d", &p, &sc, &bits);
        AURON_CHECK(n >= 2 && bits == 128, "only decimal128 is supported: " + s);
        return DType::decimal(p, sc);
    }
    fail("unsupported Arrow format string '" + s + "'");
}

std::string format_of(const DType& t) {
    switch (t.id) {
        case T_NULL: return "n";
        case T_BOOL: return "b";
        case T_INT8: return "c";
        case T_INT16: return "s";
        case T_INT32: return "i";
        case T_INT64: return "l";
        case T_FLOAT32: return "f";
        case T_FLOAT64: return "g";
        case T_UTF8: return "u";
        case T_BINARY: return "z";
        case T_DATE32: return "tdD";
        case T_DATE64: return "tdm";
        case T_TIMESTAMP: {
            const char* u = t.unit == 0 ? "s" : t.unit == 1 ? "m" : t.unit == 2 ? "u" : "n";
            return std::string("ts") + u + ":" + t.tz;
        }
        case T_DECIMAL128: return "d:" + std::to_string(t.precision) + "," + std::to_string(t.scale);
        case T_LIST: return "+l";
    }
    return "n";
}

// a field's type from its schema: a list ("+l") takes its element from the one child, which must be flat
static DType dtype_from_schema(const ArrowSchema* c) {
    AURON_CHECK(c->dictionary == nullptr, "dictionary-encoded columns are not supported");
    std::string f(c->format ? c->format : "");
    if (f == "+L" || f.rfind("+w:", 0) == 0) fail("unsupported Arrow format string '" + f + "': only 32-bit-offset lists are supported");
    if (f != "+l") return dtype_from_format(c->format);
    AURON_CHECK(c->n_children == 1 && c->children[0], "malformed Arrow list schema");
    const ArrowSchema* e = c->children[0];
    DType et = dtype_from_schema(e);
    if (et.id == T_LIST) fail("a list whose element is itself a list: nested types are out of scope");
    return DType::list(et, (e->flags & 2) != 0, e->name ? e->name : "item");
}

Schema schema_from_arrow(const ArrowSchema* s) {
    AURON_CHECK(s && s->format && std::string(s->format) == "+s", "expected a struct schema");
    Schema out;
    for (int64_t i = 0; i < s->n_children; i++) {
        const ArrowSchema* c = s->children[i];
        AURON_CHECK(c->dictionary == nullptr, "dictionary-encoded columns are not supported");
        Field f;
        f.name = c->name ? c->name : "";
        f.type = dtype_from_schema(c);
        f.nullable = (c->flags & 2) != 0;
        out.fields.push_back(f);
    }
    return out;
}

struct SchemaPriv {
    std::string format, name;
    std::vector<ArrowSchema*> children;
};
static void release_schema(ArrowSchema* s) {
    if (!s || !s->release) return;
    auto* p = static_cast<SchemaPriv*>(s->private_data);
    for (auto* c : p->children) {
        if (c->release) c->release(c);
        delete c;
    }
    delete p;
    s->release = nullptr;
}
static void fill_schema(ArrowSchema* out, const std::string& format, const std::string& name, bool nullable) {
    auto* p = new SchemaPriv;
    p->format = format;
    p->name = name;
    memset(out, 0, sizeof(*out));
    out->format = p->format.c_str();
    out->name = p->name.c_str();
    out->flags = nullable ? 2 : 0;
    out->release = release_schema;
    out->private_data = p;
}
static void fill_field_schema(ArrowSchema* c, const DType& t, const std::string& name, bool nullable) {
    fill_schema(c, format_of(t), name, nullable);
    if (t.id != T_LIST) return;
    auto* p = static_cast<SchemaPriv*>(c->private_data);
    auto* e = new ArrowSchema;
    fill_field_schema(e, *t.elem, t.elem_name, t.elem_nullable);
    p->children.push_back(e);
    c->n_children = 1;
    c->children = p->children.data();
}
void schema_to_arrow(const Schema& s, ArrowSchema* out) {
    fill_schema(out, "+s", "", false);
    auto* p = static_cast<SchemaPriv*>(out->private_data);
    for (auto& f : s.fields) {
        auto* c = new ArrowSchema;
        fill_field_schema(c, f.type, f.name, true);
        p->children.push_back(c);
    }
    out->n_children = (int64_t)p->children.size();
    out->children = p->children.data();
}

// ------------------------------------------------------------------------------------------- import
static Buf import_bits(Ctx& ctx, const uint8_t* bits, int64_t offset, int64_t len) {
    int64_t nbytes = bitmap_alloc_bytes(len);
    Buf b = dalloc_zero(ctx, nbytes);
    if (len == 0) return b;
    if ((offset & 7) == 0) {
        CUDA_OK(cudaMemcpyAsync(b->ptr, bits + offset / 8, bitmap_bytes(len), cudaMemcpyHostToDevice, ctx.stream));
    } else {
        std::vector<uint8_t> tmp(bitmap_bytes(len), 0);
        for (int64_t i = 0; i < len; i++) {
            int64_t s = offset + i;
            if ((bits[s >> 3] >> (s & 7)) & 1) tmp[i >> 3] |= (uint8_t)(1u << (i & 7));
        }
        CUDA_OK(cudaMemcpyAsync(b->ptr, tmp.data(), tmp.size(), cudaMemcpyHostToDevice, ctx.stream));
        ctx.sync();   // tmp dies here
    }
    return b;
}

static ColumnPtr import_column(Ctx& ctx, const ArrowArray* a, const DType& t) {
    auto c = std::make_shared<Column>();
    c->type = t;
    c->len = a->length;
    int64_t off = a->offset, len = a->length;
    if (t.id == T_NULL) {
        c->null_count = len;
        return c;
    }
    AURON_CHECK(a->n_buffers >= 2, "malformed Arrow array");
    const uint8_t* validity = static_cast<const uint8_t*>(a->buffers[0]);
    if (validity && a->null_count != 0) {
        c->validity = import_bits(ctx, validity, off, len);
        c->null_count = a->null_count > 0 ? a->null_count : -1;
    }
    if (t.id == T_BOOL) {
        c->data = import_bits(ctx, static_cast<const uint8_t*>(a->buffers[1]), off, len);
    } else if (t.width() > 0) {
        int w = t.width();
        c->data = dalloc(ctx, (size_t)len * w);
        if (len) CUDA_OK(cudaMemcpyAsync(c->data->ptr, static_cast<const uint8_t*>(a->buffers[1]) + off * w, (size_t)len * w, cudaMemcpyHostToDevice, ctx.stream));
    } else if (t.is_varlen()) {
        AURON_CHECK(a->n_buffers >= 3, "malformed utf8 array");
        const int32_t* offs = static_cast<const int32_t*>(a->buffers[1]);
        const uint8_t* data = static_cast<const uint8_t*>(a->buffers[2]);
        int32_t first = len ? offs[off] : 0, last = len ? offs[off + len] : 0;
        c->offsets = dalloc(ctx, (size_t)(len + 1) * 4);
        if (first == 0) {
            if (offs) CUDA_OK(cudaMemcpyAsync(c->offsets->ptr, offs + off, (size_t)(len + 1) * 4, cudaMemcpyHostToDevice, ctx.stream));
            else CUDA_OK(cudaMemsetAsync(c->offsets->ptr, 0, 4, ctx.stream));
        } else {
            std::vector<int32_t> tmp(len + 1);
            for (int64_t i = 0; i <= len; i++) tmp[i] = offs[off + i] - first;
            CUDA_OK(cudaMemcpyAsync(c->offsets->ptr, tmp.data(), tmp.size() * 4, cudaMemcpyHostToDevice, ctx.stream));
            ctx.sync();
        }
        c->data_bytes = last - first;
        c->data = dalloc(ctx, (size_t)c->data_bytes);
        if (c->data_bytes) CUDA_OK(cudaMemcpyAsync(c->data->ptr, data + first, (size_t)c->data_bytes, cudaMemcpyHostToDevice, ctx.stream));
    } else if (t.id == T_LIST) {
        // offsets rebased to start at 0; the child keeps only elements [offsets[off], offsets[off + len]) of its array
        AURON_CHECK(a->n_buffers >= 2 && a->n_children == 1 && a->children[0], "malformed Arrow list array");
        const int32_t* offs = static_cast<const int32_t*>(a->buffers[1]);
        int32_t first = len ? offs[off] : 0, last = len ? offs[off + len] : 0;
        const ArrowArray* ch = a->children[0];
        AURON_CHECK(first >= 0 && last >= first && last <= ch->length, "Arrow list offsets outside the child array");
        std::vector<int32_t> tmp((size_t)len + 1, 0);
        for (int64_t i = 0; i <= len && len; i++) {
            tmp[(size_t)i] = offs[off + i] - first;
            AURON_CHECK(i == 0 || tmp[(size_t)i] >= tmp[(size_t)i - 1], "Arrow list offsets are not monotonic");
        }
        c->offsets = dalloc(ctx, (size_t)(len + 1) * 4);
        CUDA_OK(cudaMemcpyAsync(c->offsets->ptr, tmp.data(), tmp.size() * 4, cudaMemcpyHostToDevice, ctx.stream));
        ArrowArray view = *ch;   // shallow: same buffers, the window of this slice
        view.offset += first;
        view.length = last - first;
        if (view.null_count != 0) view.null_count = -1;
        c->child = import_column(ctx, &view, *t.elem);
        ctx.sync();   // tmp dies here
    } else {
        fail("import: unsupported type " + t.str());
    }
    return c;
}

BatchPtr import_batch(Ctx& ctx, const ArrowArray* arr, const Schema& schema) {
    AURON_CHECK(arr->n_children == (int64_t)schema.fields.size(), "batch/schema column count mismatch");
    AURON_CHECK(arr->offset == 0, "sliced struct arrays are not supported at the boundary");
    auto b = std::make_shared<Batch>();
    b->num_rows = arr->length;
    for (int64_t i = 0; i < arr->n_children; i++) {
        const ArrowArray* ch = arr->children[i];
        AURON_CHECK(ch->length == arr->length, "ragged struct array");
        b->cols.push_back(import_column(ctx, ch, schema.fields[i].type));
    }
    ctx.sync();   // the caller may release / reuse the host buffers as soon as we return
    return b;
}

BatchPtr import_batch_slice(Ctx& ctx, const ArrowArray* arr, const Schema& schema, int64_t lo, int64_t len) {
    AURON_CHECK(arr->n_children == (int64_t)schema.fields.size(), "batch/schema column count mismatch");
    AURON_CHECK(arr->offset == 0 && lo >= 0 && len >= 0 && lo + len <= arr->length, "slice outside the host batch");
    auto b = std::make_shared<Batch>();
    b->num_rows = len;
    for (int64_t i = 0; i < arr->n_children; i++) {
        ArrowArray view = *arr->children[i];   // shallow: same buffers, shifted window, never released
        view.offset += lo;
        view.length = len;
        if (view.null_count != 0) view.null_count = -1;
        view.release = nullptr;
        b->cols.push_back(import_column(ctx, &view, schema.fields[(size_t)i].type));
    }
    ctx.sync();
    return b;
}

// ------------------------------------------------------------------------------------------- export
// All buffers of an exported batch live in ONE pinned block (D2H at full PCIe rate, one stream sync per batch instead of one
// pageable copy + sync per buffer); the block goes back to the pinned pool when the last array pointing into it is released
// (children may be moved out of the struct array and outlive it, so every array holds a reference).
struct PinnedBlock {
    void* p = nullptr;
    size_t cap = 0;
    size_t used = 0;
    bool pinned = false;   // small results use plain host memory (a pinned block is at least 64 MB)
    ~PinnedBlock() {
        if (p && pinned) pinned_pool().put(p, cap);
        else free(p);
    }
    void* take(size_t n) {
        void* r = (uint8_t*)p + used;
        used += (std::max<size_t>(n, 1) + 63) & ~(size_t)63;
        return r;
    }
};
struct ArrayPriv {
    std::shared_ptr<PinnedBlock> block;
    std::vector<const void*> buffers;
    std::vector<ArrowArray*> children;
};
static void release_array(ArrowArray* a) {
    if (!a || !a->release) return;
    auto* p = static_cast<ArrayPriv*>(a->private_data);
    for (auto* c : p->children) {
        if (c->release) c->release(c);
        delete c;
    }
    delete p;
    a->release = nullptr;
}
static void* host_alloc(ArrayPriv* p, size_t n) { return p->block->take(n); }
static size_t export_bytes(const Column& c) {   // upper bound of what export_column takes from the block
    auto al = [](size_t n) { return (std::max<size_t>(n, 1) + 63) & ~(size_t)63; };
    size_t n = (size_t)c.len, t = 0;
    if (c.type.id == T_NULL) return 0;
    if (c.validity) t += al(bitmap_alloc_bytes(c.len) + 8);
    if (c.type.id == T_BOOL) t += al(bitmap_alloc_bytes(c.len) + 8);
    else if (c.type.width() > 0) t += al(n * (size_t)c.type.width());
    else if (c.type.is_varlen()) t += al((n + 1) * 4) + al((size_t)c.data_bytes);
    else if (c.type.id == T_LIST) t += al((n + 1) * 4) + export_bytes(*c.child);
    return t;
}
static int64_t count_nulls(const uint8_t* bits, int64_t n) {
    int64_t set = 0;
    int64_t full = n / 8;
    for (int64_t i = 0; i < full; i++) set += __builtin_popcount(bits[i]);
    for (int64_t i = full * 8; i < n; i++) set += (bits[i >> 3] >> (i & 7)) & 1;
    return n - set;
}

static void export_column(Ctx& ctx, const Column& c, ArrowArray* out, const std::shared_ptr<PinnedBlock>& block) {
    auto* p = new ArrayPriv;
    p->block = block;
    memset(out, 0, sizeof(*out));
    out->length = c.len;
    out->release = release_array;
    out->private_data = p;
    int64_t n = c.len;
    uint8_t* hv = nullptr;
    if (c.type.id == T_NULL) {
        out->null_count = n;
        out->n_buffers = 0;
        return;
    }
    if (c.validity) {
        hv = (uint8_t*)host_alloc(p, bitmap_alloc_bytes(n) + 8);
        if (n) CUDA_OK(cudaMemcpyAsync(hv, c.validity->ptr, bitmap_bytes(n), cudaMemcpyDeviceToHost, ctx.stream));
    }
    p->buffers.push_back(hv);
    if (c.type.id == T_BOOL) {
        uint8_t* d = (uint8_t*)host_alloc(p, bitmap_alloc_bytes(n) + 8);
        if (n) CUDA_OK(cudaMemcpyAsync(d, c.data->ptr, bitmap_bytes(n), cudaMemcpyDeviceToHost, ctx.stream));
        p->buffers.push_back(d);
    } else if (c.type.width() > 0) {
        size_t bytes = (size_t)n * c.type.width();
        uint8_t* d = (uint8_t*)host_alloc(p, bytes);
        if (bytes) CUDA_OK(cudaMemcpyAsync(d, c.data->ptr, bytes, cudaMemcpyDeviceToHost, ctx.stream));
        p->buffers.push_back(d);
    } else if (c.type.is_varlen()) {
        int32_t* o = (int32_t*)host_alloc(p, (size_t)(n + 1) * 4);
        CUDA_OK(cudaMemcpyAsync(o, c.offsets->ptr, (size_t)(n + 1) * 4, cudaMemcpyDeviceToHost, ctx.stream));
        uint8_t* d = (uint8_t*)host_alloc(p, (size_t)c.data_bytes);
        if (c.data_bytes) CUDA_OK(cudaMemcpyAsync(d, c.data->ptr, (size_t)c.data_bytes, cudaMemcpyDeviceToHost, ctx.stream));
        p->buffers.push_back(o);
        p->buffers.push_back(d);
    } else if (c.type.id == T_LIST) {
        int32_t* o = (int32_t*)host_alloc(p, (size_t)(n + 1) * 4);
        CUDA_OK(cudaMemcpyAsync(o, c.offsets->ptr, (size_t)(n + 1) * 4, cudaMemcpyDeviceToHost, ctx.stream));
        p->buffers.push_back(o);
        auto* ch = new ArrowArray;
        export_column(ctx, *c.child, ch, block);
        p->children.push_back(ch);
        out->n_children = 1;
        out->children = p->children.data();
    } else {
        fail("export: unsupported type " + c.type.str());
    }
    out->null_count = hv ? -1 : 0;   // counted after the batch's single sync
    out->n_buffers = (int64_t)p->buffers.size();
    out->buffers = p->buffers.data();
}

static void fix_null_counts(ArrowArray* a) {
    if (a->null_count < 0) a->null_count = count_nulls((const uint8_t*)a->buffers[0], a->length);
    for (int64_t k = 0; k < a->n_children; k++) fix_null_counts(a->children[k]);
}

void export_batch(Ctx& ctx, const Batch& b, const Schema& schema, ArrowArray* out, size_t pinned_from) {
    AURON_CHECK(b.cols.size() == schema.fields.size(), "export: batch/schema column count mismatch");
    auto* p = new ArrayPriv;
    memset(out, 0, sizeof(*out));
    out->length = b.num_rows;
    out->null_count = 0;
    out->release = release_array;
    out->private_data = p;
    p->buffers.push_back(nullptr);
    out->n_buffers = 1;
    out->buffers = p->buffers.data();
    auto block = std::make_shared<PinnedBlock>();
    size_t total = 64;
    for (auto& c : b.cols) total += export_bytes(*c);
    if (total >= pinned_from) {
        block->p = pinned_pool().get(total, &block->cap);
        block->pinned = true;
    } else {
        if (posix_memalign(&block->p, 64, total) != 0) fail("out of host memory");
        block->cap = total;
    }
    p->block = block;
    for (auto& c : b.cols) {
        auto* ch = new ArrowArray;
        export_column(ctx, *c, ch, block);
        p->children.push_back(ch);
    }
    ctx.sync();   // one sync for every buffer of the batch
    for (size_t i = 0; i < b.cols.size(); i++) fix_null_counts(p->children[i]);
    out->n_children = (int64_t)p->children.size();
    out->children = p->children.data();
}

}  // namespace auron
