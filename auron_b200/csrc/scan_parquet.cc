// scan_parquet.cc -- ParquetScanExec: host side of the Parquet scan (row P1).  Mirrors ParquetExec::execute
// (datafusion-ext-plans/src/parquet_exec.rs:151-204), the IO adaptor (:294-467: ranged reads through
// FSDataInputWrapper.readFully) and AuronSchemaAdapter (scan/mod.rs:56-160: case-insensitive column match,
// missing columns -> NULL, INT32/INT64 decimals widened by value copy).
//
// Host work per device batch (up to AURON_GPU_CHUNK_ROWS rows, possibly spanning files):
//   1. plan   : footers (Thrift), row-group selection by file range, list of column chunks
//   2. fetch  : HBM-resident file images are used in place; host files are pread by a thread pool into one pinned
//               staging buffer and uploaded with a single async copy
//   3. parse  : page headers of every chunk (Thrift) in parallel on host threads -> page / dictionary descriptors and the list of
//               device decompression jobs (SNAPPY: k_snappy.cu, large literal chains are split into stored-copy jobs here, tags
//               only; ZSTD and LZ4_RAW: k_zstd.cu, one job per page body); the pages whose body the host must see are decompressed
//               on the host cores (nullable v1 PLAIN string pages, delta-encoded string pages, v1 list pages), UNCOMPRESSED pages
//               are decoded in place;
//               delta-encoded string pages are rewritten as PLAIN, Hive partition columns become constant columns, row groups
//               that the pruning predicates exclude by their statistics are skipped at plan time
//   4. decode : k_parquet.cu, one scout launch for all flat columns + one decode launch per column (a list column scouts its
//               element values on its own and builds its layout with k_parquet_levels.cu) -- or, when the plan above is
//               Filter -> HashAggregate of the supported shape, next_fused(): the batch goes through k_fused.cu instead and no
//               column is materialised (three batches in flight on their own stream pairs, see next_fused)
#include <dlfcn.h>
#include <fcntl.h>
#include <unistd.h>

#include <algorithm>
#include <atomic>
#include <condition_variable>
#include <deque>
#include <exception>
#include <functional>
#include <mutex>
#include <thread>

#include "../../include/auron_b200.h"
#include "operators.h"
#include "parquet_dev.h"
#include "host_pool.h"
#include "parquet_meta.h"
#include "pb.h"

namespace auron {

// ------------------------------------------------------------------------------------------ device-resident files
struct DeviceFile {
    std::vector<uint8_t> host;   // page headers / footer are parsed from the host copy
    std::shared_ptr<Ctx> ctx;    // declared before `dev`: the buffer is freed on this stream, so it must die first
    Buf dev;
};
static std::mutex g_file_mu;
static std::map<std::string, std::shared_ptr<DeviceFile>> g_dev_files;

void put_device_file(const std::string& path, const uint8_t* bytes, size_t len, int device) {
    auto f = std::make_shared<DeviceFile>();
    f->ctx = std::make_shared<Ctx>(device);
    f->host.assign(bytes, bytes + len);
    f->dev = to_device(*f->ctx, bytes, len);
    f->ctx->sync();
    std::lock_guard<std::mutex> l(g_file_mu);
    g_dev_files[path] = f;
}
void drop_device_file(const std::string& path) {
    std::lock_guard<std::mutex> l(g_file_mu);
    g_dev_files.erase(path);
}
static std::shared_ptr<DeviceFile> find_device_file(const std::string& path) {
    std::lock_guard<std::mutex> l(g_file_mu);
    auto it = g_dev_files.find(path);
    return it == g_dev_files.end() ? nullptr : it->second;
}

// host-resident file images (caller-owned, ideally pinned): the scan uploads column chunks straight from them, no pread
struct HostFile {
    const uint8_t* ptr;
    size_t len;
};
static std::map<std::string, HostFile> g_host_files;
void put_host_file(const std::string& path, const uint8_t* bytes, size_t len) {
    std::lock_guard<std::mutex> l(g_file_mu);
    g_host_files[path] = HostFile{bytes, len};
}
void drop_host_file(const std::string& path) {
    std::lock_guard<std::mutex> l(g_file_mu);
    g_host_files.erase(path);
}
static bool find_host_file(const std::string& path, HostFile* out) {
    std::lock_guard<std::mutex> l(g_file_mu);
    auto it = g_host_files.find(path);
    if (it == g_host_files.end()) return false;
    *out = it->second;
    return true;
}

// ------------------------------------------------------------------------------------------ codecs (system libs, no headers in the image)
typedef size_t (*zstd_decompress_fn)(void*, size_t, const void*, size_t);
typedef unsigned (*zstd_iserror_fn)(size_t);
typedef int (*lz4_decompress_fn)(const char*, char*, int, int);
static void host_decompress(int codec, const uint8_t* in, size_t in_len, uint8_t* out, size_t out_len) {
    if (codec == pq::CODEC_SNAPPY) {
        pq::snappy_decompress(in, in_len, out, out_len);
    } else if (codec == pq::CODEC_ZSTD) {
        static void* h = dlopen("libzstd.so.1", RTLD_NOW);
        AURON_CHECK(h, "libzstd.so.1 not available");
        static auto dec = (zstd_decompress_fn)dlsym(h, "ZSTD_decompress");
        static auto iserr = (zstd_iserror_fn)dlsym(h, "ZSTD_isError");
        size_t r = dec(out, out_len, in, in_len);
        AURON_CHECK(!iserr(r) && r == out_len, "zstd page decompression failed");
    } else if (codec == pq::CODEC_LZ4_RAW) {
        static void* h = dlopen("liblz4.so.1", RTLD_NOW);
        AURON_CHECK(h, "liblz4.so.1 not available");
        static auto dec = (lz4_decompress_fn)dlsym(h, "LZ4_decompress_safe");
        int r = dec((const char*)in, (char*)out, (int)in_len, (int)out_len);
        AURON_CHECK(r == (int)out_len, "lz4 page decompression failed");
    } else {
        fail("parquet codec " + std::to_string(codec) + " is not supported (UNCOMPRESSED, SNAPPY, ZSTD, LZ4_RAW are)");
    }
}

// ------------------------------------------------------------------------------------------ operator
struct PqFileSpec {
    std::string path;
    int64_t size = 0, range_start = -1, range_end = -1;
    std::vector<Literal> partition_values;   // Hive partition directory values, one per column of the partition schema
};
struct LeafColumn {            // one top-level field of the file (pq::walk_schema)
    int leaf_index;            // column chunk of the leaf the scan reads (lists: the element's), -1 = none
    pq::SchemaElement el;      // that leaf
    std::string name;          // the top-level field's name
    std::string path;          // the leaf's dotted path
    int shape = pq::SHAPE_FLAT;
    int max_def = 0, max_rep = 0, list_def = 0, elem_def = 0;
};

struct ParquetScanExec : Operator, FusedScanSource {
    std::string describe() const override {
        std::string o = "\"fs_resource_id\":" + json_quote(fs_id) + ",\"projection\":[";
        for (size_t i = 0; i < projection.size(); i++) o += (i ? "," : "") + std::to_string(projection[i]);
        o += "],\"files\":[";
        for (size_t i = 0; i < files.size(); i++)
            o += std::string(i ? "," : "") + "{\"path\":" + json_quote(files[i].path) + ",\"size\":" + std::to_string(files[i].size) + ",\"range\":[" +
                 std::to_string(files[i].range_start) + "," + std::to_string(files[i].range_end) + "]}";
        return o + "]";
    }
    std::vector<PqFileSpec> files;
    Schema table_schema;
    // FileScanConfig semantics (auron-planner/src/planner.rs:1415-1501): projection indices address [file columns..., partition columns...];
    // a partition column is the file's directory value repeated for every row of the file
    Schema part_schema;
    std::vector<int> projection;
    bool is_part_col(int pj) const { return pj >= (int)table_schema.fields.size(); }
    const Field& proj_field(int pj) const { return is_part_col(pj) ? part_schema.fields[(size_t)pj - table_schema.fields.size()] : table_schema.fields[(size_t)pj]; }
    // ParquetScanExecNode.pruning_predicates folded into closed intervals per table column (planner.rs:172-194: row groups whose
    // statistics cannot satisfy them are skipped; predicates of another shape prune nothing)
    std::vector<int> prune_cols;
    std::vector<int64_t> prune_lo, prune_hi;
    int64_t row_groups_pruned = 0;
    std::string fs_id;
    size_t file_pos = 0;

    // state of one opened file; kept alive for the batch that references it
    struct FileState {
        PqFileSpec spec;
        std::shared_ptr<DeviceFile> dev_file;
        HostFile host_file{nullptr, 0};   // registered host image (optional)
        int fd = -1;
        pq::FileMeta meta;
        std::vector<LeafColumn> leaves;
        std::vector<size_t> row_groups;   // selected row groups
        ~FileState() {
            if (fd >= 0) close(fd);
        }
    };
    std::shared_ptr<FileState> cur;   // currently open file
    size_t rg_pos = 0;
    void* pinned = nullptr;
    size_t pinned_cap = 0;
    unsigned host_threads = 16;

    void read_at(Task& t, FileState& f, int64_t pos, void* dst, int64_t len) {
        if (f.dev_file) {
            AURON_CHECK(pos >= 0 && (size_t)(pos + len) <= f.dev_file->host.size(), "parquet read out of range");
            memcpy(dst, f.dev_file->host.data() + pos, (size_t)len);
            return;
        }
        if (f.host_file.ptr) {
            AURON_CHECK(pos >= 0 && (size_t)(pos + len) <= f.host_file.len, "parquet read out of range");
            memcpy(dst, f.host_file.ptr + pos, (size_t)len);
            return;
        }
        if (t.cb && t.cb->read_fully) {   // FSDataInputWrapper.readFully (internal_file_reader.rs:64-68)
            int64_t got = t.cb->read_fully(t.cb->user, fs_id.c_str(), f.spec.path.c_str(), pos, dst, len);
            AURON_CHECK(got == len, "read_fully failed for " + f.spec.path);
            return;
        }
        if (f.fd < 0) {
            f.fd = open(f.spec.path.c_str(), O_RDONLY);
            AURON_CHECK(f.fd >= 0, "cannot open " + f.spec.path);
        }
        int64_t done = 0;
        while (done < len) {
            ssize_t r = pread(f.fd, (uint8_t*)dst + done, (size_t)(len - done), pos + done);
            AURON_CHECK(r > 0, "short read on " + f.spec.path);
            done += r;
        }
    }
    // Device-side landing buffers for encoded column chunks.  Plain cudaMalloc blocks recycled across batches and
    // tasks: a stream-ordered allocation made by the producer thread on the copy stream contends with the task
    // thread's own cudaMallocAsync calls inside the driver (small allocations can stall for milliseconds).
    struct DevStagePool {
        std::mutex mu;
        struct Blk {
            void* p;
            size_t cap;
            int device;
        };
        std::vector<Blk> free_list;
        void* get(size_t n, int device, size_t* cap) {
            {
                std::lock_guard<std::mutex> l(mu);
                size_t best = SIZE_MAX;
                for (size_t i = 0; i < free_list.size(); i++)
                    if (free_list[i].device == device && free_list[i].cap >= n && (best == SIZE_MAX || free_list[i].cap < free_list[best].cap)) best = i;
                if (best != SIZE_MAX) {
                    Blk e = free_list[best];
                    free_list.erase(free_list.begin() + best);
                    *cap = e.cap;
                    return e.p;
                }
            }
            void* p = nullptr;
            size_t c = std::max<size_t>(n + n / 8, 64 << 20);
            CUDA_OK(cudaMalloc(&p, c));
            *cap = c;
            return p;
        }
        void put(void* p, size_t cap, int device) {
            std::lock_guard<std::mutex> l(mu);
            free_list.push_back(Blk{p, cap, device});
            while (free_list.size() > 16) {   // keep the cache bounded: drop the smallest block
                size_t worst = 0;
                for (size_t i = 1; i < free_list.size(); i++)
                    if (free_list[i].cap < free_list[worst].cap) worst = i;
                cudaFree(free_list[worst].p);
                free_list.erase(free_list.begin() + worst);
            }
        }
    };
    static DevStagePool& dev_stage_pool() {
        static DevStagePool pool;
        return pool;
    }
    void* staging(size_t n) {
        if (n > pinned_cap) {
            if (pinned) pinned_pool().put(pinned, pinned_cap);
            pinned = pinned_pool().get(n, &pinned_cap);
        }
        return pinned;
    }
    void open_file(Task& t) {
        auto fs = std::make_shared<FileState>();
        fs->spec = files[file_pos];
        fs->dev_file = find_device_file(fs->spec.path);
        if (!fs->dev_file) find_host_file(fs->spec.path, &fs->host_file);
        int64_t size = fs->dev_file ? (int64_t)fs->dev_file->host.size() : (fs->host_file.ptr ? (int64_t)fs->host_file.len : fs->spec.size);
        AURON_CHECK(size >= 12, "not a parquet file: " + fs->spec.path);
        uint8_t tail[8];
        read_at(t, *fs, size - 8, tail, 8);
        AURON_CHECK(memcmp(tail + 4, "PAR1", 4) == 0, "missing PAR1 magic in " + fs->spec.path);
        uint32_t flen;
        memcpy(&flen, tail, 4);
        AURON_CHECK((int64_t)flen + 8 <= size, "corrupt parquet footer length");
        std::vector<uint8_t> footer(flen);
        read_at(t, *fs, size - 8 - flen, footer.data(), flen);
        fs->meta = pq::parse_file_meta(footer.data(), footer.size());
        AURON_CHECK(!fs->meta.schema.empty(), "empty parquet schema");
        // every top-level field with its shape; nested fields the query does not read cost nothing here
        const pq::SchemaTree tree = pq::walk_schema(fs->meta);
        for (const auto& tf : tree.fields) {
            LeafColumn lc;
            lc.leaf_index = -1;
            lc.el = fs->meta.schema[(size_t)tf.element];
            lc.name = tf.name;
            lc.path = tf.name;
            lc.shape = tf.shape;
            lc.list_def = tf.list_def;
            lc.elem_def = tf.elem_def;
            if (tf.leaf >= 0) {
                const pq::SchemaLeaf& l = tree.leaves[(size_t)tf.leaf];
                lc.leaf_index = l.chunk;
                lc.el = fs->meta.schema[(size_t)l.element];
                lc.path = l.path;
                lc.max_def = l.max_def;
                lc.max_rep = l.max_rep;
            }
            fs->leaves.push_back(lc);
        }
        for (int pj : projection) {   // a projected field of a shape the scan does not read fails here, with rows or without
            if (is_part_col(pj) || table_schema.fields[(size_t)pj].type.id == T_NULL) continue;
            const int li = find_leaf(*fs, table_schema.fields[(size_t)pj].name);
            if (li >= 0) check_shape(fs->leaves[(size_t)li], table_schema.fields[(size_t)pj]);
        }
        for (size_t g = 0; g < fs->meta.row_groups.size(); g++) {
            const auto& rg = fs->meta.row_groups[g];
            if (rg.columns.empty()) continue;
            int64_t start = rg.columns[0].start_offset();
            if (fs->spec.range_start >= 0 && !(start >= fs->spec.range_start && start < fs->spec.range_end)) continue;
            if (!prune_cols.empty() && row_group_pruned(*fs, rg)) {
                row_groups_pruned++;
                continue;
            }
            fs->row_groups.push_back(g);
        }
        rg_pos = 0;
        cur = fs;
    }
    struct Conv {   // a PqConv with its factor (conversion_of)
        int32_t kind = PQ_CV_COPY;
        uint64_t mul = 1, mul_hi = 0;
    };
    // can no row of this row group satisfy the pruning intervals?  (min / max statistics of INT32 / INT64 chunks; a chunk whose
    // values are all NULL satisfies no comparison)
    bool row_group_pruned(const FileState& f, const pq::RowGroup& rg) const {
        for (size_t i = 0; i < prune_cols.size(); i++) {
            const int li = find_leaf(f, table_schema.fields[(size_t)prune_cols[i]].name);
            if (li < 0 || f.leaves[(size_t)li].shape != pq::SHAPE_FLAT) continue;   // (list statistics bound the elements, not the rows)
            const int leaf_index = f.leaves[(size_t)li].leaf_index;
            if ((size_t)leaf_index >= rg.columns.size()) continue;
            const pq::ColumnMeta& cm = rg.columns[(size_t)leaf_index];
            const pq::Statistics& st = cm.stats;
            if (st.has_null_count && st.null_count == cm.num_values && cm.num_values > 0) return true;
            const pq::SchemaElement& el = f.leaves[(size_t)li].el;
            Conv cv;   // (a column the table cannot read fails when it is projected, not here)
            if (!try_conversion(el, table_schema.fields[(size_t)prune_cols[i]].type, &cv)) continue;
            int64_t mn, mx;   // bounds in the table's type: the pruning intervals are
            if (!converted_bounds(el, cv, st, &mn, &mx)) continue;
            if (mx < prune_lo[i] || mn > prune_hi[i]) return true;
        }
        return false;
    }
    static int find_leaf(const FileState& f, const std::string& name) {
        for (size_t i = 0; i < f.leaves.size(); i++)
            if (f.leaves[i].name == name) return (int)i;
        for (size_t i = 0; i < f.leaves.size(); i++) {   // case-insensitive (scan/mod.rs:56-100)
            const std::string& n = f.leaves[i].name;
            if (n.size() != name.size()) continue;
            bool eq = true;
            for (size_t k = 0; k < n.size(); k++) eq = eq && tolower(n[k]) == tolower(name[k]);
            if (eq) return (int)i;
        }
        return -1;
    }
    // layout signature of a file for the projected columns; a batch never mixes different layouts
    std::string signature(const FileState& f) const {
        std::string s;
        for (int pj : projection) {
            if (is_part_col(pj)) {
                s += "P;";
                continue;
            }
            int li = find_leaf(f, table_schema.fields[pj].name);
            if (li < 0 || table_schema.fields[pj].type.id == T_NULL) s += "-;";
            else {
                const LeafColumn& lc = f.leaves[li];
                const pq::SchemaElement& el = lc.el;   // (the annotation decides the conversion; a list's levels its layout)
                s += std::to_string(lc.shape) + ":" + std::to_string(lc.max_def) + ":" + std::to_string(lc.list_def) + ":" + std::to_string(lc.elem_def) + ":" +
                     std::to_string(f.leaves[li].leaf_index) + ":" + std::to_string(el.type) + ":" + std::to_string(el.repetition) + ":" + std::to_string(el.type_length) +
                     ":" + std::to_string(el.logical) + ":" + std::to_string(el.ts_unit) + ":" + std::to_string(el.int_bits) + ":" + std::to_string(el.int_signed) + ":" +
                     std::to_string(el.precision) + ":" + std::to_string(el.scale) + ";";
            }
        }
        return s;
    }

    // descriptors of one column chunk (local numbering; rebased when merged into the column's lists)
    struct ChunkPages {
        std::vector<PqPage> pages;
        std::vector<PqDict> dicts;
        std::vector<PqByteSection> secs;
        int64_t value_table_size = 0;
        // compressed chunks: page payloads decompressed here, pointers patched after the upload
        std::vector<uint8_t> unc;
        struct Fix {
            size_t page;   // index into pages, or SIZE_MAX for a dictionary
            size_t dict, sec;
            int64_t off;
            bool dev;      // off is relative to the device scratch (decompressed by the GPU), else to `unc` (decompressed here)
        };
        std::vector<Fix> fixes;
        // SNAPPY, ZSTD and LZ4_RAW pages are decompressed on the device (all but the pages the host must see): jobs with dst as an OFFSET into a scratch
        // buffer of gpu_unc_bytes that the task thread allocates; `fixes` then patch the descriptors with the scratch base
        std::vector<PqDecompJob> jobs;
        bool snappy_jobs = true;   // jobs for k_snappy.cu, else for k_zstd.cu (ZSTD / LZ4_RAW chunks)
        int64_t gpu_unc_bytes = 0;
        int64_t pages_dev = 0, pages_host = 0;   // compressed pages (dictionary and data) decompressed on the device / on the host
        bool has_v1_inline = false;
        bool has_delta = false;   // some pages are DELTA_BINARY_PACKED: transcribed to PLAIN in the scratch buffer (pq_delta_to_plain)
        // list columns: the level sections of every data page (slot_start local to the chunk; pointers of pages decompressed here are
        // offsets into `unc` where levels_in_unc says so), and the chunk's level slots and non-null values
        std::vector<PqLevelPage> levels;
        std::vector<uint8_t> levels_in_unc;
        int64_t n_slots = 0, n_vals = 0;
    };
    struct ChunkTask {
        std::shared_ptr<FileState> file;
        const pq::ColumnMeta* cm = nullptr;
        int col = 0;               // index into projection
        int64_t row_start = 0;
        const uint8_t* host = nullptr;
        const uint8_t* dev = nullptr;
        int64_t stage_off = -1;    // offset in the pinned staging buffer (files that must be pread)
        int64_t dev_off = -1;      // offset in the batch's device buffer (every chunk that is uploaded)
        ChunkPages out;
    };
    struct FileSeg {
        size_t file;         // index into files
        int64_t row0, rows;
    };
    struct ColState {
        int leaf = -1;   // index into leaves, -1 = missing
        int part_col = -1;   // >= 0: column of the partition schema (no file column at all)
        pq::SchemaElement el;
        bool is_string = false;
        Conv cv;   // physical value -> table type
        std::vector<PqPage> pages;
        std::vector<PqDict> dicts;
        std::vector<PqByteSection> secs;
        int64_t value_table_size = 0;
        std::vector<Buf> keep;
        bool has_v1_inline = false;   // some v1 pages still need their level / value sections split on the device
        bool has_delta = false;
        // bounds of the non-null values from the column-chunk statistics of every chunk in the batch (INT32 / INT64)
        bool stat_ok = true;
        int64_t stat_min = INT64_MAX, stat_max = INT64_MIN;
        // the leaf's levels; a one-level list (shape SHAPE_LIST) decodes its element values as a required column of n_vals values
        // (pages[].row_start = first value of the page) and its layout from `levels`
        int shape = pq::SHAPE_FLAT;
        int max_def = 0, max_rep = 0, list_def = 0, elem_def = 0;
        std::string path;
        std::vector<PqLevelPage> levels;
        int64_t n_slots = 0, n_vals = 0;
    };

    // `p[0, n)` is a Snappy block of `unc` bytes made of exactly one literal element: returns the offset of the literal's
    // bytes (> 0), else 0
    static int64_t snappy_single_literal(const uint8_t* p, int64_t n, int64_t unc) {
        int64_t i = 0;
        uint64_t v = 0;
        for (int shift = 0; shift <= 28; shift += 7) {
            if (i >= n) return 0;
            uint8_t b = p[i++];
            v |= (uint64_t)(b & 0x7f) << shift;
            if (!(b & 0x80)) break;
            if (shift == 28) return 0;
        }
        if ((int64_t)v != unc || i >= n || unc <= 0) return 0;
        const uint8_t tag = p[i++];
        if (tag & 3) return 0;
        int64_t len = (tag >> 2) + 1;
        if (len > 60) {
            const int nb = (int)len - 60;
            if (i + nb > n) return 0;
            uint32_t w = 0;
            for (int k = 0; k < nb; k++) w |= (uint32_t)p[i + k] << (8 * k);
            i += nb;
            len = (int64_t)w + 1;
        }
        return (len == unc && i + len == n) ? i : 0;
    }
    // (the tag walk of a Snappy block, pq::snappy_split, and the host decoders of the delta string encodings and of level streams live
    // in parquet_meta.cc, where auron_b200_parquet_describe exercises them on the CPU)
    static bool gpu_snappy() {
        return getenv("AURON_HOST_SNAPPY") == nullptr;   // AURON_HOST_SNAPPY=1: decompress on the host cores instead
    }
    // pure CPU: walk the pages of one column chunk (thread-safe, no CUDA calls)
    static int bit_width(int v) {
        int b = 0;
        while ((1 << b) <= v) b++;
        return b;
    }
    static void parse_chunk(ChunkTask& ct, const ColState& cs) {
        const pq::SchemaElement& el = cs.el;
        const bool is_string = cs.is_string;
        const pq::ColumnMeta& cm = *ct.cm;
        ChunkPages& out = ct.out;
        const uint8_t* host = ct.host;
        const uint8_t* dev = ct.dev;
        const int64_t len = cm.total_compressed;
        const bool is_list = cs.shape == pq::SHAPE_LIST;
        const int max_def = is_list ? cs.max_def : el.repetition == 1 ? 1 : 0;
        out.snappy_jobs = cm.codec == pq::CODEC_SNAPPY;
        const bool compressed = cm.codec != pq::CODEC_UNCOMPRESSED;
        // SNAPPY, ZSTD and LZ4_RAW bodies are decompressed on the device (k_snappy.cu, k_zstd.cu) unless the host needs them
        const bool dev_codec = (cm.codec == pq::CODEC_SNAPPY && gpu_snappy()) || cm.codec == pq::CODEC_ZSTD || cm.codec == pq::CODEC_LZ4_RAW;
        int64_t pos = 0, values_seen = 0, rows = is_list ? 0 : ct.row_start;   // (lists: rows counts values)
        int cur_dict = -1;
        while (pos < len && values_seen < cm.num_values) {
            pq::PageHeader h = pq::parse_page_header(host + pos, (size_t)(len - pos));
            const uint8_t* payload_h = host + pos + h.header_len;
            const uint8_t* payload_d = dev + pos + h.header_len;
            AURON_CHECK(h.compressed_size >= 0 && h.uncompressed_size >= 0 && h.num_values >= 0, "corrupt parquet page header (negative size)");
            AURON_CHECK(pos + h.header_len + h.compressed_size <= len, "parquet page overruns its column chunk");
            pos += h.header_len + h.compressed_size;
            if (h.type == pq::PAGE_INDEX) continue;
            int64_t unc_off = -1;
            int32_t lvl_bytes = h.type == pq::PAGE_DATA_V2 ? h.def_bytes + h.rep_bytes : 0;
            const bool page_compressed = compressed && !(h.type == pq::PAGE_DATA_V2 && !h.v2_compressed);
            // Where the page body ends up: in place (uncompressed, or "stored" below), decompressed on the device, or decompressed
            // on the host (AURON_HOST_SNAPPY; and the pages whose body the host must see: a PLAIN string page needs its non-null count
            // to place its values, which a nullable v1 page only has inside its body; delta strings are rewritten here).
            const bool delta_strings = is_string && (h.encoding == pq::ENC_DELTA_LENGTH_BYTE_ARRAY || h.encoding == pq::ENC_DELTA_BYTE_ARRAY);
            // (the levels of a v1 list page are inside its body: the host counts the page's values from them, so it decompresses the body)
            const bool page_dev = dev_codec && !(is_string && h.type == pq::PAGE_DATA && h.encoding == pq::ENC_PLAIN && max_def > 0) && !delta_strings &&
                                  !(is_list && h.type == pq::PAGE_DATA);
            bool on_device = false;
            int64_t gap = 0;   // stored v2 page with level sections: Snappy framing bytes between the levels and the values
            if (page_compressed) (page_dev ? out.pages_dev : out.pages_host)++;
            if (page_compressed && page_dev && cm.codec != pq::CODEC_SNAPPY) {
                AURON_CHECK(h.uncompressed_size >= lvl_bytes && h.compressed_size >= lvl_bytes, "corrupt parquet page sizes");
                on_device = true;
            } else if (page_compressed && page_dev) {
                AURON_CHECK(h.uncompressed_size >= lvl_bytes && h.compressed_size >= lvl_bytes, "corrupt parquet page sizes");
                // Incompressible pages (bit-packed dictionary indices of random keys) are one Snappy literal: preamble, literal
                // tag, raw body.  The body is then already in HBM inside the chunk, a few bytes further on: no job, no copy.
                const int64_t lit = snappy_single_literal(payload_h + lvl_bytes, h.compressed_size - lvl_bytes, h.uncompressed_size - lvl_bytes);
                if (lit > 0 && lvl_bytes == 0) {
                    payload_h += lit;
                    payload_d += lit;
                } else if (lit > 0) {
                    gap = lit;
                } else {
                    on_device = true;
                }
            }
            if (on_device) {
                unc_off = out.gpu_unc_bytes;
                out.gpu_unc_bytes += ((int64_t)h.uncompressed_size + 8 + 15) & ~(int64_t)15;
                if (lvl_bytes) out.jobs.push_back(PqDecompJob{payload_d, (uint8_t*)(intptr_t)unc_off, lvl_bytes, lvl_bytes, 0, 0});   // v2 levels are stored
                // A large incompressible body (an 816 KB dictionary of surrogate keys, a 1 MB page of bit-packed indices) is a
                // chain of 64 KB literals, in a nullable v1 data page behind a few back references that compress the level bytes:
                // one warp walking the chain serially was the long pole of the whole launch, however few pages
                // the batch holds.  The host walks the tags (16 per MB); the literals behind the last back reference
                // become independent stored-copy jobs of <= 16 KB, the elements before them a short Snappy job of their own.
                // Not split: a body whose tail is ONE literal in a nullable v1 page (the decoder leaves that one in place), and
                // bodies of many elements (compressible data: the walk stops after 4096 tags).
                std::vector<pq::LitPiece> pieces;
                const bool v1_nullable = h.type == pq::PAGE_DATA && max_def > 0;
                const uint8_t* body_h = payload_h + lvl_bytes;
                const uint8_t* body_d = payload_d + lvl_bytes;
                const int64_t body_in = h.compressed_size - lvl_bytes, body_out = h.uncompressed_size - lvl_bytes;
                int64_t head_in = 0, head_out = 0;
                if (cm.codec != pq::CODEC_SNAPPY) {   // one job per page body: ZSTD frames or one LZ4 block
                    out.jobs.push_back(PqDecompJob{body_d, (uint8_t*)(intptr_t)(unc_off + lvl_bytes), (int32_t)body_in, (int32_t)body_out,
                                                   cm.codec == pq::CODEC_ZSTD ? PQ_JOB_ZSTD : PQ_JOB_LZ4, 0});
                } else if (body_out > (64 << 10) && pq::snappy_split(body_h, body_in, body_out, 4096, &head_in, &head_out, &pieces) &&
                    body_out - head_out >= (32 << 10) && !(v1_nullable && pieces.size() == 1)) {
                    int64_t dst = unc_off + lvl_bytes;
                    if (head_out > 0)   // kind 2: the preamble states the length of the whole body, the job ends after head_out bytes
                        out.jobs.push_back(PqDecompJob{body_d, (uint8_t*)(intptr_t)dst, (int32_t)head_in, (int32_t)head_out, 2, v1_nullable ? 1 : 0});
                    dst += head_out;
                    for (auto& pc : pieces) {
                        for (int64_t o = 0; o < pc.len; o += 16 << 10) {
                            const int32_t l = (int32_t)std::min<int64_t>(16 << 10, pc.len - o);
                            out.jobs.push_back(PqDecompJob{body_d + pc.src_off + o, (uint8_t*)(intptr_t)(dst + o), l, l, 0, 0});
                        }
                        dst += pc.len;
                    }
                } else {
                    out.jobs.push_back(PqDecompJob{body_d, (uint8_t*)(intptr_t)(unc_off + lvl_bytes), (int32_t)body_in, (int32_t)body_out, 1, 0});
                }
                payload_h = nullptr;
            } else if (page_compressed && !page_dev) {
                unc_off = (int64_t)out.unc.size();
                out.unc.resize(out.unc.size() + (size_t)h.uncompressed_size + 8);
                if (lvl_bytes) memcpy(out.unc.data() + unc_off, payload_h, (size_t)lvl_bytes);   // v2 levels are never compressed
                host_decompress(cm.codec, payload_h + lvl_bytes, (size_t)(h.compressed_size - lvl_bytes), out.unc.data() + unc_off + lvl_bytes,
                                (size_t)(h.uncompressed_size - lvl_bytes));
                payload_h = nullptr;
            }
            auto hp = [&](int64_t o) -> const uint8_t* { return unc_off >= 0 ? out.unc.data() + unc_off + o : payload_h + o; };
            if (h.type == pq::PAGE_DICTIONARY) {
                AURON_CHECK(h.encoding == pq::ENC_PLAIN || h.encoding == pq::ENC_PLAIN_DICTIONARY, "unsupported dictionary page encoding");
                PqDict d{payload_d, h.num_values, (int32_t)out.value_table_size};
                cur_dict = (int)out.dicts.size();
                out.dicts.push_back(d);
                size_t sec_idx = SIZE_MAX;
                if (is_string) {
                    sec_idx = out.secs.size();
                    out.secs.push_back({payload_d, h.uncompressed_size, h.num_values, (int32_t)out.value_table_size});
                    out.value_table_size += h.num_values;
                }
                if (unc_off >= 0) out.fixes.push_back({SIZE_MAX, (size_t)cur_dict, sec_idx, unc_off, on_device});
                continue;
            }
            AURON_CHECK(h.type == pq::PAGE_DATA || h.type == pq::PAGE_DATA_V2, "unknown parquet page type");
            PqPage pg;
            memset(&pg, 0, sizeof(pg));
            pg.job = -1;
            pg.num_values = h.num_values;
            pg.row_start = (int32_t)rows;
            pg.encoding = h.encoding;
            pg.dict_id = cur_dict;
            const bool delta_ints = h.encoding == pq::ENC_DELTA_BINARY_PACKED && (el.type == pq::PT_INT32 || el.type == pq::PT_INT64);
            AURON_CHECK(h.encoding == pq::ENC_PLAIN || ((h.encoding == pq::ENC_RLE_DICTIONARY || h.encoding == pq::ENC_PLAIN_DICTIONARY) && cur_dict >= 0) ||
                            (h.encoding == pq::ENC_RLE && el.type == pq::PT_BOOLEAN) || delta_ints || delta_strings,
                        "parquet encoding " + std::to_string(h.encoding) + (h.encoding == 9 ? " (BYTE_STREAM_SPLIT)" : "") + " of column " + el.name +
                            " is not supported (PLAIN, RLE_DICTIONARY, RLE booleans and the DELTA encodings are)");
            if (delta_ints) {   // transcribed on the device, after the sections of the page are known (pq_delta_to_plain)
                pg.encoding = pq::ENC_PLAIN;
                pg.delta_dst16 = (int32_t)(out.gpu_unc_bytes / 16) + 1;
                out.gpu_unc_bytes += ((int64_t)h.num_values * (el.type == pq::PT_INT32 ? 4 : 8) + 16 + 15) & ~(int64_t)15;
                out.has_delta = true;
            }
            int64_t o = 0, total = h.uncompressed_size;
            int32_t delta_nn = -1;   // non-null values of a delta-encoded string page (its streams say so)
            int32_t list_nn = -1;    // list pages: the page's non-null values
            int64_t rep_off = 0, def_off = 0;   // list pages: level sections (offsets in the page body)
            PqLevelPage lv{};
            if (is_list) {
                lv.n_slots = h.num_values;
                if (h.type == pq::PAGE_DATA) {   // [u32 length][repetition levels][u32 length][definition levels][values]
                    AURON_CHECK(h.rep_encoding == pq::ENC_RLE && h.def_encoding == pq::ENC_RLE, "only RLE repetition and definition levels are supported (column " + cs.path + ")");
                    uint32_t rl = 0, dl = 0;
                    AURON_CHECK(total >= 8, "corrupt parquet list page (column " + cs.path + ")");
                    memcpy(&rl, hp(0), 4);
                    AURON_CHECK((int64_t)rl + 8 <= total, "corrupt parquet list page levels (column " + cs.path + ")");
                    memcpy(&dl, hp(4 + (int64_t)rl), 4);
                    AURON_CHECK((int64_t)rl + 8 + (int64_t)dl <= total, "corrupt parquet list page levels (column " + cs.path + ")");
                    rep_off = 4;
                    def_off = 8 + (int64_t)rl;
                    lv.rep_len = (int32_t)rl;
                    lv.def_len = (int32_t)dl;
                    o = def_off + dl;
                    list_nn = (int32_t)pq::hybrid_count(hp(def_off), dl, bit_width(max_def), h.num_values, (uint32_t)max_def);
                } else {   // v2: levels stored uncompressed in front of the values, the header counts the NULL slots
                    AURON_CHECK(h.rep_bytes >= 0 && h.def_bytes >= 0 && (int64_t)h.rep_bytes + h.def_bytes <= total && h.num_nulls >= 0 && h.num_nulls <= h.num_values,
                                "corrupt parquet list page levels (column " + cs.path + ")");
                    def_off = h.rep_bytes;
                    lv.rep_len = h.rep_bytes;
                    lv.def_len = h.def_bytes;
                    o = (int64_t)h.rep_bytes + h.def_bytes;
                    list_nn = h.num_values - h.num_nulls;
                }
            } else if (h.type == pq::PAGE_DATA) {
                if (max_def > 0) {
                    AURON_CHECK(h.def_encoding == pq::ENC_RLE, "only RLE definition levels are supported");
                    pg.def_ptr = (const uint8_t*)(intptr_t)4;   // offsets now, pointers once the base is known
                    if (on_device) {
                        // the length word is inside the compressed body: pq_fix_v1_pages splits the sections on the device
                        AURON_CHECK(total >= 4, "corrupt parquet page");
                        pg.def_len = -1;
                        pg.job = (int32_t)out.jobs.size() - 1;   // the Snappy job pushed for this page above
                        if (out.jobs.back().kind == 1) out.jobs.back().v1_levels = 1;   // (a split body has its flag already)
                        out.has_v1_inline = true;
                    } else {
                        uint32_t dl;
                        memcpy(&dl, hp(0), 4);
                        pg.def_len = (int32_t)dl;
                        o = 4 + dl;
                    }
                }
            } else {
                o = h.rep_bytes;
                if (max_def > 0 && h.def_bytes > 0) {
                    pg.def_ptr = (const uint8_t*)(intptr_t)o;
                    pg.def_len = h.def_bytes;
                }
                if (max_def > 0 && h.def_bytes == 0 && h.num_nulls == h.num_values) pg.all_null = 1;
                o += h.def_bytes;
            }
            AURON_CHECK(o <= total, "corrupt parquet page levels");
            if (delta_strings) {   // (never on_device: the body is on the host, in the file image or in out.unc)
                const std::vector<uint8_t> head(hp(0), hp(0) + o);
                int32_t nn = 0;
                const std::vector<uint8_t> plain = pq::delta_strings_to_plain(hp(o + gap), (size_t)(total - o - gap), h.encoding == pq::ENC_DELTA_BYTE_ARRAY, &nn, (size_t)h.num_values);
                AURON_CHECK(list_nn < 0 || nn == list_nn, "corrupt parquet list page: its values do not match its levels (column " + cs.path + ")");
                unc_off = (int64_t)out.unc.size();
                out.unc.resize(out.unc.size() + head.size() + plain.size() + 8);
                if (!head.empty()) memcpy(out.unc.data() + unc_off, head.data(), head.size());
                if (!plain.empty()) memcpy(out.unc.data() + unc_off + o, plain.data(), plain.size());
                total = o + (int64_t)plain.size();
                gap = 0;
                pg.encoding = pq::ENC_PLAIN;
                delta_nn = nn;
            }
            int64_t val_off = o + gap;
            pg.val_len = (int32_t)(total - o);   // v1 inline: the whole body until the device splits it
            const uint8_t* base_d = unc_off >= 0 ? nullptr : payload_d;
            if (base_d) {
                pg.def_ptr = pg.def_len ? base_d + (intptr_t)pg.def_ptr : nullptr;   // (def_len -1 never reaches here: on_device => no base yet)
                pg.val_ptr = base_d + val_off;
            } else {
                pg.val_ptr = (const uint8_t*)(intptr_t)val_off;
            }
            size_t sec_idx = SIZE_MAX;
            if (is_string && pg.encoding == pq::ENC_PLAIN) {
                // PLAIN string pages need their exact non-null count: v2 gives it, v1 requires the def levels (whose section, behind the
                // length word, lies inside the page: o <= total above)
                int32_t nn = delta_nn >= 0 ? delta_nn : list_nn >= 0 ? list_nn : h.type == pq::PAGE_DATA_V2 ? h.num_values - h.num_nulls : max_def == 0 ? h.num_values
                           : (int32_t)pq::hybrid_count(hp(4), (size_t)pg.def_len, 1, h.num_values, 1);
                pg.plain_value_base = (int32_t)out.value_table_size;
                sec_idx = out.secs.size();
                out.secs.push_back({base_d ? pg.val_ptr : nullptr, pg.val_len, nn, (int32_t)out.value_table_size});
                out.value_table_size += nn;
            }
            if (is_list) {
                // the values decode as a required column: the page holds list_nn of them, placed behind those of the pages before it
                pg.num_values = list_nn;
                // v2 levels are never compressed: they are read where the chunk lies; v1 levels from the page body, in place or in `unc`
                const bool in_unc = h.type == pq::PAGE_DATA && unc_off >= 0;
                const uint8_t* lbase = in_unc ? (const uint8_t*)(intptr_t)unc_off : h.type == pq::PAGE_DATA ? payload_d : dev + (pos - h.compressed_size);
                lv.rep = lbase + rep_off;
                lv.def = lbase + def_off;
                lv.slot_start = (int32_t)out.n_slots;
                AURON_CHECK(out.n_slots + h.num_values <= (int64_t)INT32_MAX, "parquet list column " + cs.path + ": a column chunk of more than 2^31 - 1 level slots");
                out.levels.push_back(lv);
                out.levels_in_unc.push_back(in_unc ? 1 : 0);
                out.n_slots += h.num_values;
                out.n_vals += list_nn;
            }
            if (unc_off >= 0) out.fixes.push_back({out.pages.size(), 0, sec_idx, unc_off, on_device});
            out.pages.push_back(pg);
            rows += is_list ? list_nn : h.num_values;
            values_seen += h.num_values;
        }
    }

    // the column state of a projected field that the file holds: its shape must be one the table type can read
    static void check_shape(const LeafColumn& lc, const Field& fld) {
        const bool want_list = fld.type.id == T_LIST;
        if (lc.shape == pq::SHAPE_FLAT && want_list)
            fail("cannot read parquet column " + lc.name + " (a primitive column, physical type " + std::to_string(lc.el.type) + ") as " + fld.type.str());
        if (lc.shape == pq::SHAPE_LIST && !want_list)
            fail("cannot read parquet column " + lc.name + " (a list of physical type " + std::to_string(lc.el.type) + ") as " + fld.type.str());
        if (lc.shape != pq::SHAPE_FLAT && lc.shape != pq::SHAPE_LIST)
            fail("cannot read parquet column " + lc.name + " (a " + pq::shape_name(lc.shape) + "): only primitive columns and lists of primitives are read");
    }
    static void setup_column(ColState& cs, const LeafColumn& lc, const Field& fld) {
        check_shape(lc, fld);
        AURON_CHECK(lc.leaf_index >= 0, "parquet column " + lc.name + " has no leaf");
        cs.el = lc.el;
        cs.shape = lc.shape;
        cs.path = lc.path;
        cs.max_def = lc.max_def;
        cs.max_rep = lc.max_rep;
        cs.list_def = lc.list_def;
        cs.elem_def = lc.elem_def;
        if (lc.shape == pq::SHAPE_LIST) {
            AURON_CHECK(fld.type.elem && fld.type.elem->id != T_LIST, "list column " + fld.name + " without a flat element type");
            AURON_CHECK(lc.max_rep == 1 && lc.max_def >= lc.elem_def && lc.max_def <= lc.elem_def + 1, "parquet column " + lc.name + ": unexpected list levels");
            pq::SchemaElement e = lc.el;
            e.name = lc.path;   // (a conversion error names the column and its element)
            cs.cv = conversion_of(e, *fld.type.elem);
        } else {
            cs.cv = conversion_of(lc.el, fld.type);
        }
        cs.is_string = lc.el.type == pq::PT_BYTE_ARRAY;
    }

    static int phys_width(int phys, int type_length) {
        switch (phys) {
            case pq::PT_INT32: case pq::PT_FLOAT: return 4;
            case pq::PT_INT64: case pq::PT_DOUBLE: return 8;
            case pq::PT_FLBA: return type_length;
            case pq::PT_INT96: return 12;
            default: return 0;
        }
    }
    // ---- one conversion per column: (physical type, annotation, table type) -> PqConv.  The reference reads the file's Arrow type
    // and AuronSchemaAdapter (scan/mod.rs:103-160) casts it to the table's; the pairs below are those whose cast is exact, plus the
    // integer -> decimal value copy of scan/mod.rs:131-136.  Everything else fails (DESIGN section 4, "Parquet column conversions").
    // false for a pair outside the table
    static bool try_conversion(const pq::SchemaElement& el, const DType& t, Conv* out) {
        Conv cv;
        bool ok = false;
        auto kind = [&](int32_t k) {
            cv.kind = k;
            ok = true;
        };
        const int lk = el.logical;
        const bool is_int_target = t.id == T_INT8 || t.id == T_INT16 || t.id == T_INT32 || t.id == T_INT64;
        if (lk == pq::LK_DECIMAL) {
            // decimal(p1, s1) -> decimal(p2, s2): x 10^(s2 - s1) when no digit is lost and the integer part fits (always exact)
            const bool storage = (el.type == pq::PT_INT32 && el.precision <= 9) || (el.type == pq::PT_INT64 && el.precision <= 18) ||
                                 (el.type == pq::PT_FLBA && el.type_length >= 1 && el.type_length <= 16);
            if (storage && t.id == T_DECIMAL128 && el.precision >= 1 && el.scale >= 0 && t.scale >= el.scale && t.precision - t.scale >= el.precision - el.scale) {
                unsigned __int128 m = 1;
                for (int i = el.scale; i < t.scale; i++) m *= 10;
                kind(m == 1 ? PQ_CV_SEXT : PQ_CV_DEC);   // (at its own scale: the value copy)
                cv.mul = (uint64_t)m;
                cv.mul_hi = (uint64_t)(m >> 64);
            }
        } else {
            switch (el.type) {
                case pq::PT_BOOLEAN: if (t.id == T_BOOL && lk == pq::LK_NONE) kind(PQ_CV_COPY); break;
                case pq::PT_INT32: {
                    const bool sgn = lk == pq::LK_NONE || (lk == pq::LK_INTEGER && el.int_signed && el.int_bits <= 32);
                    const int bits = lk == pq::LK_INTEGER ? el.int_bits : 32;
                    if (lk == pq::LK_INTEGER && !el.int_signed && el.int_bits <= 32) {
                        if (is_int_target && 8 * t.width() > bits) kind(PQ_CV_ZEXT);   // UINT_n into a strictly wider signed integer
                    } else if (sgn || lk == pq::LK_DATE) {
                        if ((t.id == T_INT8 || t.id == T_INT16) && sgn && bits <= 8 * t.width()) kind(PQ_CV_COPY);
                        else if (t.id == T_INT32 || t.id == T_DATE32) kind(PQ_CV_COPY);
                        else if (t.id == T_INT64) kind(PQ_CV_SEXT);
                        else if (t.id == T_FLOAT64 && sgn) kind(PQ_CV_I32_F64);
                        else if (t.id == T_DECIMAL128 && sgn) kind(PQ_CV_SEXT);
                    }
                    break;
                }
                case pq::PT_INT64:
                    if (lk == pq::LK_TIMESTAMP) {
                        if (t.id == T_INT64) kind(PQ_CV_COPY);   // the stored count, as arrow casts a timestamp to int64
                        else if (t.id == T_TIMESTAMP && t.unit >= 0 && t.unit <= 3) {
                            const int d = t.unit - el.ts_unit;
                            uint64_t m = 1;
                            for (int i = 0; i < 3 * (d < 0 ? -d : d); i++) m *= 10;
                            kind(d == 0 ? PQ_CV_COPY : d > 0 ? PQ_CV_TS_MUL : PQ_CV_TS_DIV);
                            cv.mul = m;
                        }
                    } else if (lk == pq::LK_NONE || (lk == pq::LK_INTEGER && el.int_signed)) {
                        if (t.id == T_INT64 || t.id == T_DATE64 || t.id == T_TIMESTAMP) kind(PQ_CV_COPY);   // (a plain int64 is a count in the table's unit)
                        else if (t.id == T_DECIMAL128) kind(PQ_CV_SEXT);
                    }
                    break;
                case pq::PT_INT96: if (t.id == T_TIMESTAMP) kind(PQ_CV_COPY); break;   // Spark's legacy timestamp encoding (parquet_exec.rs:192 coerces it)
                case pq::PT_FLOAT: if (t.id == T_FLOAT32) kind(PQ_CV_COPY); else if (t.id == T_FLOAT64) kind(PQ_CV_F32_F64); break;
                case pq::PT_DOUBLE: if (t.id == T_FLOAT64) kind(PQ_CV_COPY); break;
                case pq::PT_BYTE_ARRAY: if (t.is_varlen()) kind(PQ_CV_COPY); break;
                default: break;
            }
        }
        *out = cv;
        return ok;
    }
    static Conv conversion_of(const pq::SchemaElement& el, const DType& t) {
        Conv cv;
        if (try_conversion(el, t, &cv)) return cv;
        const int lk = el.logical;
        static const char* kLogical[] = {"", ", STRING", ", DECIMAL", ", DATE", ", TIMESTAMP", ", INTEGER", ", other annotation"};
        std::string ann = kLogical[lk >= 0 && lk <= 6 ? lk : 6];
        if (lk == pq::LK_DECIMAL) ann += "(" + std::to_string(el.precision) + "," + std::to_string(el.scale) + ")";
        if (lk == pq::LK_INTEGER) ann += std::string("(") + std::to_string(el.int_bits) + (el.int_signed ? ",signed)" : ",unsigned)");
        if (lk == pq::LK_TIMESTAMP) ann += el.ts_unit == 1 ? "(ms)" : el.ts_unit == 2 ? "(us)" : "(ns)";
        fail("cannot read parquet column " + el.name + " (physical type " + std::to_string(el.type) + ann + ") as " + t.str());
    }
    // Column-chunk min / max in the table's type (Statistics.min_value / max_value are PLAIN-encoded: little-endian two's complement).
    // False when they do not bound the converted values (no statistics, or a conversion that is not monotone into an integer).
    static bool converted_bounds(const pq::SchemaElement& el, const Conv& cv, const pq::Statistics& st, int64_t* mn, int64_t* mx) {
        const size_t w = el.type == pq::PT_INT32 ? 4 : el.type == pq::PT_INT64 ? 8 : 0;
        if (!w || !st.has_min || !st.has_max || st.min_value.size() != w || st.max_value.size() != w) return false;
        auto read = [&](const std::string& s) -> int64_t {
            if (w == 8) {
                int64_t v;
                memcpy(&v, s.data(), 8);
                return v;
            }
            uint32_t v;
            memcpy(&v, s.data(), 4);
            return cv.kind == PQ_CV_ZEXT ? (int64_t)v : (int64_t)(int32_t)v;   // an unsigned column's statistics are unsigned
        };
        int64_t a = read(st.min_value), b = read(st.max_value);
        switch (cv.kind) {
            case PQ_CV_COPY: case PQ_CV_SEXT: case PQ_CV_ZEXT: break;
            case PQ_CV_TS_MUL: {   // a bound whose product leaves int64 is dropped: those values are NULL after the conversion
                const int64_t m = (int64_t)cv.mul;
                a = a < INT64_MIN / m ? INT64_MIN : a > INT64_MAX / m ? INT64_MAX : a * m;
                b = b > INT64_MAX / m ? INT64_MAX : b < INT64_MIN / m ? INT64_MIN : b * m;
                break;
            }
            case PQ_CV_TS_DIV: a /= (int64_t)cv.mul, b /= (int64_t)cv.mul; break;   // truncation is monotone
            default: return false;
        }
        *mn = a;
        *mx = b;
        return true;
    }

    const PqDecompResult* decomp_results = nullptr;   // results of the current batch's decompression launch (device)
    uint8_t* unc_scratch_ptr = nullptr;               // the current batch's scratch buffer and status word (device)
    int32_t* status_ptr = nullptr;
    // The device copies of a column's page and dictionary descriptors, fixed up for the decoders on `ctx` in this order: the level /
    // value sections of v1 pages decompressed on the device (pq_fix_v1_pages), then the PLAIN transcription of DELTA_BINARY_PACKED
    // pages into the batch's scratch buffer (pq_delta_to_plain)
    struct ColDescriptors {
        Buf pages, dicts;
    };
    ColDescriptors upload_descriptors(Ctx& ctx, const ColState& cs) const {
        ColDescriptors d;
        d.pages = to_device(ctx, cs.pages.empty() ? (const void*)"" : (const void*)cs.pages.data(), cs.pages.size() * sizeof(PqPage));
        d.dicts = to_device(ctx, cs.dicts.empty() ? (const void*)"" : (const void*)cs.dicts.data(), cs.dicts.size() * sizeof(PqDict));
        if (cs.has_v1_inline) pq_fix_v1_pages(ctx, P<PqPage>(d.pages), (int)cs.pages.size(), decomp_results);
        if (cs.has_delta) pq_delta_to_plain(ctx, P<PqPage>(d.pages), (int)cs.pages.size(), unc_scratch_ptr, cs.el.type == pq::PT_INT32 ? 4 : 8, status_ptr);
        return d;
    }
    // decode arguments of a column whose values are read as type `t` (a list column: its element type); the caller sets the mode
    // and the outputs
    static PqColumnArgs column_args(const ColState& cs, const ColDescriptors& d, const DType& t, int max_def) {
        PqColumnArgs a;
        memset(&a, 0, sizeof(a));
        a.pages = P<PqPage>(d.pages);
        a.dicts = P<PqDict>(d.dicts);
        a.n_pages = (int)cs.pages.size();
        a.phys_type = cs.el.type;
        a.type_length = cs.el.type_length;
        a.phys_width = phys_width(cs.el.type, cs.el.type_length);
        a.out_type = t.id;
        a.out_width = t.width();
        a.out_unit = t.unit;
        a.conv = cs.cv.kind;
        a.conv_mul = cs.cv.mul;
        a.conv_mul_hi = cs.cv.mul_hi;
        a.max_def = max_def;
        return a;
    }
    // side streams ("lanes") of the fused path, see next_fused
    std::vector<std::unique_ptr<Ctx>> lanes;
    std::vector<int> lane_priority;
    // Lane contexts (a stream + its staged-upload arena) outlive the scan that used them: every task is a new ParquetScanExec, and six
    // stream creations / destructions per task are host time inside a step of a few milliseconds; idle lanes wait in a process-wide pool instead
    // (which also keeps the stream-ordered allocator's per-stream caches warm).
    struct LanePool {
        std::mutex mu;
        struct Idle {
            std::unique_ptr<Ctx> ctx;
            int device, priority;
        };
        std::vector<Idle> idle;
        std::unique_ptr<Ctx> take(int device, int priority) {
            {
                std::lock_guard<std::mutex> g(mu);
                for (size_t i = 0; i < idle.size(); i++)
                    if (idle[i].device == device && idle[i].priority == priority) {
                        std::unique_ptr<Ctx> c = std::move(idle[i].ctx);
                        idle.erase(idle.begin() + (long)i);
                        return c;
                    }
            }
            return std::unique_ptr<Ctx>(new Ctx(device, priority));
        }
        void give(std::unique_ptr<Ctx> c, int priority) {
            if (!c || !c->stream) return;
            try {
                c->sync();   // idle by now (the scan has retired its batches); also recycles the lane's staged-upload arena
            } catch (...) {
                return;      // (called from a destructor: a stream in an error state is simply not kept)
            }
            c->prof.clear();
            c->kernel_launches = 0;
            std::lock_guard<std::mutex> g(mu);
            if (idle.size() < 24) idle.push_back(Idle{std::move(c), 0, priority}), idle.back().device = idle.back().ctx->device;
        }
    };
    static LanePool& lane_pool() {
        static LanePool* p = new LanePool();   // (never destroyed: streams must not be torn down after the CUDA runtime at process exit)
        return *p;
    }
    Ctx& lane(Task& t, int i, int priority = 0) {
        while ((int)lanes.size() <= i) {
            lanes.push_back(lane_pool().take(t.ctx.device, priority));
            lanes.back()->profile = t.ctx.profile;
            lane_priority.push_back(priority);
        }
        return *lanes[(size_t)i];
    }
    static void chain(cudaStream_t from, cudaStream_t to) {   // work queued on `to` from here on runs after everything queued on `from` so far
        cudaEvent_t e;
        CUDA_OK(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
        CUDA_OK(cudaEventRecord(e, from));
        CUDA_OK(cudaStreamWaitEvent(to, e, 0));
        CUDA_OK(cudaEventDestroy(e));
    }
    void fold_lanes(Task& t) {   // profile entries and launch counts of the lanes belong to the task
        for (auto& l : lanes) {
            for (auto& e : l->prof) t.ctx.prof.push_back(e);
            l->prof.clear();
            t.ctx.kernel_launches += l->kernel_launches;
            l->kernel_launches = 0;
        }
    }
    // every row a NULL list: zero offsets, a clear validity bitmap and an empty child of the element type (a file without the column)
    static ColumnPtr null_list_column(Ctx& ctx, const DType& t, int64_t n_rows) {
        auto col = std::make_shared<Column>();
        col->type = t;
        col->len = n_rows;
        col->offsets = dalloc_zero(ctx, (size_t)(n_rows + 1) * 4);
        col->validity = dalloc_zero(ctx, bitmap_alloc_bytes(n_rows));
        col->null_count = n_rows;
        col->child = make_column(ctx, *t.elem, 0, false);
        return col;
    }
    // A one-level list column of the batch (on the task stream): the element values of every page decode as one required column,
    // the level pass (k_parquet_levels.cu) gives the offsets, the list validity and each element's value, one gather places the values.
    ColumnPtr build_list_column(Task& t, ColState& cs, const Field& fld, int64_t n_rows) {
        const DType& et = *fld.type.elem;
        const int64_t nv = cs.n_vals;
        AURON_CHECK(nv <= cs.n_slots, "corrupt parquet list column " + cs.path + ": more values than level slots");
        const ColDescriptors d = upload_descriptors(t.ctx, cs);
        PqColumnArgs a = column_args(cs, d, et, 0);   // (the values of a list page have no gaps)
        ColumnPtr vals;   // fixed-width: the values; strings: the value table, gathered once through str_idx below
        Buf str_idx;      // strings: value -> entry of the value table
        if (cs.is_string) {
            vals = pq_build_value_table(t.ctx, cs.secs, cs.value_table_size, et);
            str_idx = dalloc(t.ctx, (size_t)std::max<int64_t>(nv, 1) * 4);
            a.mode = PQ_MODE_INDEX;
            a.out_idx = P<int32_t>(str_idx);
            if (!cs.pages.empty()) pq_decode_pages(t.ctx, a, cs.pages);
        } else {
            vals = std::make_shared<Column>();
            vals->type = et;
            vals->len = nv;
            vals->data = et.id == T_BOOL ? dalloc_zero(t.ctx, bitmap_alloc_bytes(nv)) : dalloc(t.ctx, (size_t)std::max<int64_t>(nv, 1) * et.width());
            if (cs.cv.kind == PQ_CV_TS_MUL) {   // (overflowing products are NULL)
                vals->validity = dalloc_zero(t.ctx, bitmap_alloc_bytes(nv));
                vals->null_count = -1;
            }
            a.mode = PQ_MODE_VALUES;
            a.out = vals->data->ptr;
            a.out_valid = P<uint32_t>(vals->validity);
            if (!cs.pages.empty()) pq_decode_pages(t.ctx, a, cs.pages);
        }
        PqListShape sh;
        sh.rep_bw = bit_width(cs.max_rep);
        sh.def_bw = bit_width(cs.max_def);
        sh.list_def = cs.list_def;
        sh.elem_def = cs.elem_def;
        sh.max_def = cs.max_def;
        auto col = std::make_shared<Column>();
        col->type = fld.type;
        col->len = n_rows;
        col->offsets = dalloc(t.ctx, (size_t)(n_rows + 1) * 4);
        if (cs.list_def > 0) {
            col->validity = dalloc_zero(t.ctx, bitmap_alloc_bytes(n_rows));
            col->null_count = -1;
        }
        Buf elem_idx = dalloc(t.ctx, (size_t)std::max<int64_t>(cs.n_slots, 1) * 4);
        Buf counts = dalloc(t.ctx, 4 * sizeof(int64_t));
        Buf dlevels = to_device(t.ctx, cs.levels.empty() ? (const void*)"" : (const void*)cs.levels.data(), cs.levels.size() * sizeof(PqLevelPage));
        pq_list_levels(t.ctx, P<PqLevelPage>(dlevels), (int)cs.levels.size(), cs.n_slots, n_rows, sh, P<int32_t>(col->offsets), P<uint32_t>(col->validity),
                       P<int32_t>(elem_idx), P<int64_t>(counts));
        int64_t c[4];
        to_host(t.ctx, c, counts->ptr, sizeof(c));   // (the element count sizes the gather)
        AURON_CHECK(c[3] == 0, "corrupt parquet list column " + cs.path + ": malformed levels in page " + std::to_string(c[3] - 1) + " of the batch");
        AURON_CHECK(c[0] == n_rows && c[2] == nv, "corrupt parquet list column " + cs.path + ": the levels hold " + std::to_string(c[0]) + " rows and " +
                                                       std::to_string(c[2]) + " values, the pages " + std::to_string(n_rows) + " and " + std::to_string(nv));
        if (str_idx) pq_compose_index(t.ctx, P<int32_t>(elem_idx), P<int32_t>(str_idx), c[1]);   // element -> value-table entry
        col->child = take(t.ctx, *vals, P<int32_t>(elem_idx), c[1], cs.max_def > cs.elem_def);
        return col;
    }
    BatchPtr build_batch(Task& t, std::vector<ColState>& cols, int64_t n_rows, const std::vector<FileSeg>& file_segs) {
        AURON_CHECK(n_rows < (int64_t)INT32_MAX, "parquet batch too large");
        auto out = std::make_shared<Batch>();
        out->num_rows = n_rows;
        // One scout launch for all flat columns of the batch (a column alone is a few thousand page-warps, too few for 132 SMs):
        // the per-column work is prepared in the loop, scouted together, then decoded column by column.
        struct Pending {
            size_t out_pos;
            PqPrepared pr;
            ColumnPtr table;   // strings: value table to gather from after the index decode
            Buf idx;
            ColDescriptors descr;
            bool nullable;
        };
        std::vector<Pending> pending;
        for (size_t ci = 0; ci < projection.size(); ci++) {
            const Field& fld = proj_field(projection[ci]);
            ColState& cs = cols[ci];
            if (cs.part_col >= 0) {   // Hive partition column: the directory value of each file, repeated for its rows
                std::vector<ColumnPtr> pieces;
                for (auto& fsg : file_segs) {
                    const auto& pv = files[fsg.file].partition_values;
                    AURON_CHECK((size_t)cs.part_col < pv.size(), "PartitionedFile carries fewer partition values than the partition schema has columns");
                    auto le = std::make_shared<Expr>();
                    le->kind = E_LITERAL;
                    le->lit = pv[(size_t)cs.part_col];
                    ExprPtr e = le;
                    if (le->lit.type != fld.type) {   // the literal's Arrow type may differ from the declared column type (e.g. int32 vs date32)
                        auto c = std::make_shared<Expr>();
                        c->kind = E_TRY_CAST;
                        c->type = fld.type;
                        c->children.push_back(le);
                        e = c;
                    }
                    Batch dummy;
                    dummy.num_rows = fsg.rows;
                    VmProgram prog = compile_projection({e}, Schema());
                    pieces.push_back(eval_projection(t.ctx, prog, dummy, nullptr, fsg.rows)[0]);
                }
                out->cols.push_back(pieces.size() == 1 ? pieces[0] : concat_columns(t.ctx, pieces));
                continue;
            }
            if (cs.leaf < 0) {   // missing column -> NULL (scan/mod.rs:84-100)
                if (fld.type.id == T_LIST) {
                    out->cols.push_back(null_list_column(t.ctx, fld.type, n_rows));
                } else if (fld.type.is_varlen()) {
                    auto c = make_column(t.ctx, fld.type, n_rows, true);
                    c->null_count = n_rows;
                    CUDA_OK(cudaMemsetAsync(c->offsets->ptr, 0, (size_t)(n_rows + 1) * 4, t.ctx.stream));
                    out->cols.push_back(c);
                } else out->cols.push_back(make_null_column(t.ctx, fld.type, n_rows));
                continue;
            }
            if (cs.shape == pq::SHAPE_LIST) {
                out->cols.push_back(build_list_column(t, cs, fld, n_rows));
                continue;
            }
            const int max_def = cs.el.repetition == 1 ? 1 : 0;
            ColumnPtr col;
            Buf validity;
            if (!cs.is_string) {
                if (max_def > 0 || cs.cv.kind == PQ_CV_TS_MUL) validity = dalloc_zero(t.ctx, bitmap_alloc_bytes(n_rows));   // (overflowing products are NULL)
                col = std::make_shared<Column>();
                col->type = fld.type;
                col->len = n_rows;
                if (fld.type.id == T_BOOL) col->data = dalloc_zero(t.ctx, bitmap_alloc_bytes(n_rows));
                else col->data = dalloc(t.ctx, (size_t)n_rows * fld.type.width());
            }
            const ColDescriptors d = upload_descriptors(t.ctx, cs);
            PqColumnArgs a = column_args(cs, d, fld.type, max_def);
            if (cs.is_string) {
                ColumnPtr table = pq_build_value_table(t.ctx, cs.secs, cs.value_table_size, fld.type);
                Buf idx = dalloc(t.ctx, (size_t)std::max<int64_t>(n_rows, 1) * 4);
                a.mode = PQ_MODE_INDEX;
                a.out_idx = P<int32_t>(idx);
                pending.push_back(Pending{out->cols.size(), pq_prepare(t.ctx, a, cs.pages), table, idx, d, max_def > 0});   // (col: the take below)
            } else {
                a.mode = PQ_MODE_VALUES;
                a.out = col->data->ptr;
                a.out_valid = P<uint32_t>(validity);
                pending.push_back(Pending{out->cols.size(), pq_prepare(t.ctx, a, cs.pages), nullptr, nullptr, d, false});
                if (validity) {
                    col->validity = validity;
                    col->null_count = -1;
                }
                const TypeId ot = fld.type.id;
                if (cs.stat_ok && cs.stat_min <= cs.stat_max && (ot == T_INT32 || ot == T_INT64 || ot == T_DATE32)) {
                    col->has_range = true;
                    col->range_min = cs.stat_min;
                    col->range_max = cs.stat_max;
                }
            }
            out->cols.push_back(col);
        }
        if (!pending.empty()) {
            std::vector<PqPrepared*> prs;
            for (auto& pd : pending) prs.push_back(&pd.pr);
            pq_scout_many(t.ctx, prs);
            for (auto& pd : pending) {
                pq_decode_prepared(t.ctx, pd.pr);
                if (pd.table) out->cols[pd.out_pos] = take(t.ctx, *pd.table, P<int32_t>(pd.idx), n_rows, pd.nullable);
            }
            pending.clear();
        }
        for (auto& l : lanes) chain(l->stream, t.ctx.stream);   // the batch is complete once every lane is
        fold_lanes(t);
        t.ctx.sync();   // chunk buffers die with `cols`
        return out;
    }

    // ---- batch pipeline: a producer thread plans, reads, uploads (copy stream) and parses up to `prefetch_depth`
    // batches ahead; the task thread merges + decodes them on the task stream.  While the GPU decodes batch k and the
    // downstream operators consume it, later batches are already crossing PCIe, so the e2e transfer hides behind
    // compute and the copy engine never waits for the task thread.
    struct Prepared {
        std::vector<ColState> cols;
        std::vector<ChunkTask> tasks;
        int64_t rows = 0, stage_bytes = 0, dev_bytes = 0;
        std::vector<FileSeg> file_segs;   // which rows of the batch come from which file (partition column values)
        void* pinned = nullptr;
        size_t pinned_cap = 0;
        void* dev = nullptr;   // from dev_stage_pool()
        void* unc_dev = nullptr;   // scratch for pages decompressed / transcribed on the device, from dev_stage_pool() (a fresh
        size_t unc_cap = 0;        // stream-ordered allocation of this size grows the driver's pool now and then, a stall of the step)
        int unc_device = 0;
        size_t dev_cap = 0;
        int device = 0;
        cudaEvent_t copied = nullptr, copy_begin = nullptr;
        int64_t fetch_ns = 0, parse_ns = 0;
    };
    cudaStream_t copy_stream = nullptr;
    int prefetch_depth = 3;
    std::thread producer;
    std::mutex qmu;
    std::condition_variable qcv;
    std::deque<std::unique_ptr<Prepared>> ready_q;
    bool producer_started = false, producer_done = false, stop_producer = false;
    std::string producer_err;

    void release(Prepared& p) {
        if (p.pinned) pinned_pool().put(p.pinned, p.pinned_cap);
        p.pinned = nullptr;
        if (p.dev) {
            // every reader of the landing buffer has finished on the normal path (build_batch ends with a stream sync);
            // on error paths make sure the uploads themselves are done before the block is recycled
            if (p.copied) cudaEventSynchronize(p.copied);
            dev_stage_pool().put(p.dev, p.dev_cap, p.device);
            p.dev = nullptr;
        }
        if (p.unc_dev) {   // (released with the batch: every kernel that read it has finished, see above)
            dev_stage_pool().put(p.unc_dev, p.unc_cap, p.unc_device);
            p.unc_dev = nullptr;
        }
        if (p.copied) cudaEventDestroy(p.copied);
        if (p.copy_begin) cudaEventDestroy(p.copy_begin);
        p.copied = p.copy_begin = nullptr;
    }

    std::unique_ptr<Prepared> plan_batch(Task& t) {
        auto pp = std::make_unique<Prepared>();
        Prepared& p = *pp;
        std::string batch_sig;
        bool started = false;
        for (;;) {
            if (file_pos >= files.size()) break;
            if (!cur) open_file(t);
            if (rg_pos >= cur->row_groups.size()) {
                cur.reset();
                file_pos++;
                continue;
            }
            const auto& rg = cur->meta.row_groups[cur->row_groups[rg_pos]];
            std::string sig = signature(*cur);
            if (started && (sig != batch_sig || p.rows + rg.num_rows > t.ctx.gpu_chunk_rows)) break;
            if (!started) {
                started = true;
                batch_sig = sig;
                p.cols.assign(projection.size(), ColState());
                for (size_t ci = 0; ci < projection.size(); ci++) {
                    if (is_part_col(projection[ci])) {
                        p.cols[ci].part_col = projection[ci] - (int)table_schema.fields.size();
                        continue;
                    }
                    const Field& fld = table_schema.fields[projection[ci]];
                    int li = find_leaf(*cur, fld.name);
                    if (fld.type.id == T_NULL) li = -1;   // a field the query does not read (NullType): NULL, whatever the file holds
                    p.cols[ci].leaf = li;
                    if (li < 0) continue;
                    setup_column(p.cols[ci], cur->leaves[(size_t)li], fld);
                }
            }
            for (size_t ci = 0; ci < projection.size(); ci++) {
                if (p.cols[ci].leaf < 0) continue;
                // (by name in THIS file: field positions differ between files whose signatures match)
                const int li = find_leaf(*cur, table_schema.fields[projection[ci]].name);
                AURON_CHECK(li >= 0, "parquet column " + table_schema.fields[projection[ci]].name + " missing from a row group of its batch");
                int leaf_index = cur->leaves[(size_t)li].leaf_index;
                AURON_CHECK((size_t)leaf_index < rg.columns.size(), "row group misses a column chunk");
                ChunkTask ct;
                ct.file = cur;
                ct.cm = &rg.columns[leaf_index];
                ct.col = (int)ci;
                ct.row_start = p.rows;
                p.tasks.push_back(std::move(ct));
            }
            if (!p.file_segs.empty() && p.file_segs.back().file == file_pos) p.file_segs.back().rows += rg.num_rows;
            else p.file_segs.push_back(FileSeg{file_pos, p.rows, rg.num_rows});
            p.rows += rg.num_rows;
            rg_pos++;
        }
        if (!started) return nullptr;
        // chunk placement: HBM-resident images in place, host files into one pinned staging buffer + one device buffer
        for (auto& ct : p.tasks) {
            int64_t start = ct.cm->start_offset(), len = ct.cm->total_compressed;
            if (ct.file->dev_file) {
                AURON_CHECK(start >= 0 && (size_t)(start + len) <= ct.file->dev_file->host.size(), "column chunk outside the file image");
                ct.host = ct.file->dev_file->host.data() + start;
                ct.dev = P<uint8_t>(ct.file->dev_file->dev) + start;
            } else {
                ct.dev_off = p.dev_bytes;
                p.dev_bytes += (len + 63) & ~(int64_t)63;
                if (ct.file->host_file.ptr) {
                    AURON_CHECK(start >= 0 && (size_t)(start + len) <= ct.file->host_file.len, "column chunk outside the host image");
                    ct.host = ct.file->host_file.ptr + start;
                } else {
                    ct.stage_off = p.stage_bytes;
                    p.stage_bytes += (len + 63) & ~(int64_t)63;
                }
            }
        }
        if (p.dev_bytes > 0) {
            if (p.stage_bytes > 0) p.pinned = pinned_pool().get((size_t)p.stage_bytes + 64, &p.pinned_cap);
            if (!copy_stream) CUDA_OK(cudaStreamCreateWithFlags(&copy_stream, cudaStreamNonBlocking));
            p.device = t.ctx.device;
            p.dev = dev_stage_pool().get((size_t)p.dev_bytes + 128, p.device, &p.dev_cap);
            CUDA_OK(cudaEventCreateWithFlags(&p.copied, t.ctx.profile ? cudaEventDefault : cudaEventDisableTiming));
            if (t.ctx.profile) CUDA_OK(cudaEventCreate(&p.copy_begin));
            for (auto& ct : p.tasks)
                if (ct.dev_off >= 0) {
                    if (ct.stage_off >= 0) ct.host = (uint8_t*)p.pinned + ct.stage_off;
                    ct.dev = (const uint8_t*)p.dev + ct.dev_off;
                }
        }
        return pp;
    }

    // read + upload + parse one planned batch
    void fetch_and_parse(Task& t, Prepared& p) {
        auto t0 = std::chrono::steady_clock::now();
        const bool via_callback = t.cb && t.cb->read_fully;
        if (p.dev_bytes > 0) {
            const int device = t.ctx.device;
            cudaSetDevice(device);
            cudaStream_t cs = copy_stream;
            if (p.copy_begin) CUDA_OK(cudaEventRecord(p.copy_begin, cs));
            // chunks that already sit in a host image need no worker: issue their uploads right away, in order
            for (auto& ct : p.tasks)
                if (ct.dev_off >= 0 && ct.stage_off < 0)
                    CUDA_OK(cudaMemcpyAsync(const_cast<uint8_t*>(ct.dev), ct.host, (size_t)ct.cm->total_compressed, cudaMemcpyHostToDevice, cs));
            // everything else is read in 4 MB slices by the worker pool (a batch may hold fewer column chunks than
            // workers); each slice is uploaded as soon as its bytes are in the pinned staging buffer
            struct Slice {
                ChunkTask* ct;
                int64_t off, len;
            };
            std::vector<Slice> slices;
            // a host runtime that cannot take upcalls from other threads gets one read per chunk on the task thread
            const bool serial_cb = via_callback && !t.cb->upcalls_from_any_thread;
            const int64_t kSlice = serial_cb ? INT64_MAX : (4 << 20);
            if (p.stage_bytes > 0)
                for (auto& ct : p.tasks) {
                    if (ct.dev_off < 0 || ct.stage_off < 0) continue;
                    for (int64_t o = 0; o < ct.cm->total_compressed; o += std::min(kSlice, ct.cm->total_compressed - o))
                        slices.push_back(Slice{&ct, o, std::min(kSlice, ct.cm->total_compressed - o)});
                }
            parallel_for(slices.size(), serial_cb ? 1 : host_threads, [&](size_t i) {
                const Slice& sl = slices[i];
                ChunkTask& ct = *sl.ct;
                int64_t start = ct.cm->start_offset() + sl.off, len = sl.len;
                uint8_t* dst = const_cast<uint8_t*>(ct.host) + sl.off;
                if (via_callback) {
                    read_at(t, *ct.file, start, dst, len);
                } else {
                    int fd = open(ct.file->spec.path.c_str(), O_RDONLY);   // own descriptor per worker read
                    AURON_CHECK(fd >= 0, "cannot open " + ct.file->spec.path);
                    int64_t done = 0;
                    while (done < len) {
                        ssize_t r = pread(fd, dst + done, (size_t)(len - done), start + done);
                        if (r <= 0) {
                            close(fd);
                            fail("short read on " + ct.file->spec.path);
                        }
                        done += r;
                    }
                    close(fd);
                }
                cudaSetDevice(device);
                cudaError_t e = cudaMemcpyAsync(const_cast<uint8_t*>(ct.dev) + sl.off, dst, (size_t)len, cudaMemcpyHostToDevice, cs);
                if (e != cudaSuccess) fail(std::string("H2D copy failed: ") + cudaGetErrorString(e));
            });
            CUDA_OK(cudaEventRecord(p.copied, copy_stream));
        }
        auto t1 = std::chrono::steady_clock::now();
        parallel_for(p.tasks.size(), host_threads, [&](size_t i) { parse_chunk(p.tasks[i], p.cols[p.tasks[i].col]); });
        auto t2 = std::chrono::steady_clock::now();
        p.fetch_ns = std::chrono::duration_cast<std::chrono::nanoseconds>(t1 - t0).count();
        p.parse_ns = std::chrono::duration_cast<std::chrono::nanoseconds>(t2 - t1).count();
    }
    void producer_loop(Task& t) {
        try {
            CUDA_OK(cudaSetDevice(t.ctx.device));
            for (;;) {
                {
                    std::unique_lock<std::mutex> l(qmu);
                    qcv.wait(l, [&] { return stop_producer || (int)ready_q.size() < prefetch_depth; });
                    if (stop_producer) break;
                }
                auto p = plan_batch(t);
                if (!p) break;
                try {
                    fetch_and_parse(t, *p);
                } catch (...) {
                    release(*p);
                    throw;
                }
                std::lock_guard<std::mutex> l(qmu);
                ready_q.push_back(std::move(p));
                qcv.notify_all();
            }
        } catch (const std::exception& e) {
            std::lock_guard<std::mutex> l(qmu);
            producer_err = e.what();
        } catch (...) {
            std::lock_guard<std::mutex> l(qmu);
            producer_err = "unknown failure in the scan prefetch thread";
        }
        std::lock_guard<std::mutex> l(qmu);
        producer_done = true;
        qcv.notify_all();
    }
    void stop() {
        if (producer.joinable()) {
            {
                std::lock_guard<std::mutex> l(qmu);
                stop_producer = true;
                qcv.notify_all();
            }
            producer.join();
        }
        for (auto& p : ready_q) release(*p);
        ready_q.clear();
    }

    ~ParquetScanExec() override {
        for (auto& f : inflight) {   // fused batches still running: their landing buffers go back only once the kernels are done
            cudaEventSynchronize(f->done);
            cudaEventDestroy(f->done);
            release(*f->sg.ready);
        }
        inflight.clear();
        stop();
        for (size_t i = 0; i < lanes.size(); i++) lane_pool().give(std::move(lanes[i]), lane_priority[i]);
        lanes.clear();
        if (copy_stream) {
            cudaStreamSynchronize(copy_stream);
            cudaStreamDestroy(copy_stream);
        }
    }

    // next planned + fetched + parsed batch, or nullptr at the end of the scan
    std::unique_ptr<Prepared> take_ready(Task& t) {
        const bool serial_cb = t.cb && t.cb->read_fully && !t.cb->upcalls_from_any_thread;
        if (serial_cb || prefetch_depth <= 0) {   // such callbacks re-enter the host runtime: stay on the task thread
            auto p = plan_batch(t);
            if (p) {
                try {
                    fetch_and_parse(t, *p);
                } catch (...) {
                    release(*p);
                    throw;
                }
            }
            return p;
        }
        if (!producer_started) {
            producer_started = true;
            producer = std::thread([this, &t] { producer_loop(t); });
        }
        std::unique_lock<std::mutex> l(qmu);
        qcv.wait(l, [&] { return !ready_q.empty() || producer_done; });
        if (ready_q.empty()) {
            if (!producer_err.empty()) fail(producer_err);
            return nullptr;
        }
        auto p = std::move(ready_q.front());
        ready_q.pop_front();
        qcv.notify_all();
        return p;
    }

    // One batch taken from the prefetch pipeline with its descriptors merged and its page decompression queued
    struct Staged {
        std::unique_ptr<Prepared> ready;
        Buf status;            // page decompression status word (device)
        bool has_jobs = false;
        std::vector<int8_t> job_codec;   // codec of every decompression job, for the error message
    };
    // nullptr ready = end of the scan
    // `wc`: the context (stream) the batch's device work is queued on -- the task's own, or one of the two lanes the fused path alternates between
    Staged stage_next(Task& t, Ctx& wc) {
        Staged sg;
        AURON_CHECK(t.is_running(), "task killed");
        std::unique_ptr<Prepared> ready;
        {
            OpTimer tw(metrics, "wait_fetch_ns");
            ready = take_ready(t);
        }
        if (!ready) {
            if (row_groups_pruned) {
                metrics.add("row_groups_pruned", row_groups_pruned);
                row_groups_pruned = 0;
            }
            return sg;
        }
        struct Guard {   // an exception below must not leak the landing buffers
            ParquetScanExec* op;
            std::unique_ptr<Prepared>* p;
            int exc;
            ~Guard() {
                if (std::uncaught_exceptions() > exc && *p) op->release(**p);
            }
        } guard{this, &ready, std::uncaught_exceptions()};
        metrics.add("fetch_ns", ready->fetch_ns);
        metrics.add("parse_ns", ready->parse_ns);
        if (ready->dev_bytes) {
            metrics.add("h2d_bytes", ready->dev_bytes);
            CUDA_OK(cudaStreamWaitEvent(wc.stream, ready->copied, 0));
        }
        Prepared& p = *ready;
        // ordered merge, rebasing dictionary ids / value-table positions; compressed chunks upload their payloads first
        std::vector<PqDecompJob> decomp_jobs;
        OpTimer* tmerge = new OpTimer(metrics, "merge_ns");
        // Phase A (serial, cheap): slot of every chunk in the per-column descriptor arrays, in the batch's scratch buffer for
        // device-decompressed pages and in the job list; value bounds from the chunk statistics.
        struct Slot {
            int64_t unc_off = 0;
            int64_t val_base = 0;   // list columns: the chunk's first value within the batch
            size_t job_base = 0, page_base = 0, dict_base = 0, sec_base = 0;
            int32_t vbase = 0;
            Buf host_unc;   // chunks decompressed on the host: their payload, uploaded below
        };
        std::vector<Slot> slots(p.tasks.size());
        int64_t unc_total = 0, pages_dev = 0, pages_host = 0;
        size_t n_jobs = 0, n_other_jobs = 0;   // Snappy jobs first, then the ZSTD / LZ4_RAW chunks' jobs (pq_decompress)
        std::vector<size_t> npages(p.cols.size(), 0), ndicts(p.cols.size(), 0), nsecs(p.cols.size(), 0);
        for (size_t ti = 0; ti < p.tasks.size(); ti++) {
            ChunkTask& ct = p.tasks[ti];
            ColState& cs = p.cols[ct.col];
            ChunkPages& cp = ct.out;
            Slot& sl = slots[ti];
            sl.unc_off = unc_total;
            unc_total += (cp.gpu_unc_bytes + 255) & ~(int64_t)255;
            if (cp.snappy_jobs) {
                sl.job_base = n_jobs;
                n_jobs += cp.jobs.size();
            } else {
                sl.job_base = n_other_jobs;   // rebased behind the Snappy jobs below
                n_other_jobs += cp.jobs.size();
            }
            pages_dev += cp.pages_dev;
            pages_host += cp.pages_host;
            sl.page_base = npages[ct.col];
            sl.dict_base = ndicts[ct.col];
            sl.sec_base = nsecs[ct.col];
            sl.vbase = (int32_t)cs.value_table_size;
            npages[ct.col] += cp.pages.size();
            ndicts[ct.col] += cp.dicts.size();
            nsecs[ct.col] += cp.secs.size();
            cs.value_table_size += cp.value_table_size;
            if (cp.gpu_unc_bytes > 0) {
                cs.has_v1_inline = cs.has_v1_inline || cp.has_v1_inline;
                cs.has_delta = cs.has_delta || cp.has_delta;
            }
            {   // statistics -> bounds of the converted values
                const pq::Statistics& st = ct.cm->stats;
                int64_t mn, mx;
                if (converted_bounds(cs.el, cs.cv, st, &mn, &mx)) {
                    cs.stat_min = std::min(cs.stat_min, mn);
                    cs.stat_max = std::max(cs.stat_max, mx);
                } else if (!(st.has_null_count && st.null_count == ct.cm->num_values)) {
                    cs.stat_ok = false;   // (an all-NULL chunk has no min / max and constrains nothing)
                }
            }
            if (!cp.unc.empty()) {   // host-decompressed payloads (ZSTD / LZ4_RAW pages, nullable v1 PLAIN string pages) are uploaded here
                sl.host_unc = to_device(wc, cp.unc.data(), cp.unc.size());
                cs.keep.push_back(sl.host_unc);
            }
            if (cs.shape == pq::SHAPE_LIST) {   // level sections, rebased to the batch (a few descriptors per page: serial)
                AURON_CHECK(cs.n_slots + cp.n_slots <= (int64_t)INT32_MAX,
                            "parquet list column " + cs.path + ": a batch of more than 2^31 - 1 list elements and empty or NULL lists; lower AURON_GPU_CHUNK_ROWS");
                sl.val_base = cs.n_vals;
                for (size_t i = 0; i < cp.levels.size(); i++) {
                    PqLevelPage lv = cp.levels[i];
                    lv.slot_start += (int32_t)cs.n_slots;
                    if (cp.levels_in_unc[i]) {
                        lv.rep = P<uint8_t>(sl.host_unc) + (intptr_t)lv.rep;
                        lv.def = P<uint8_t>(sl.host_unc) + (intptr_t)lv.def;
                    }
                    cs.levels.push_back(lv);
                }
                cs.n_slots += cp.n_slots;
                cs.n_vals += cp.n_vals;
            }
        }
        for (size_t ti = 0; ti < p.tasks.size(); ti++)
            if (!p.tasks[ti].out.snappy_jobs) slots[ti].job_base += n_jobs;
        const size_t n_snappy_jobs = n_jobs;
        n_jobs += n_other_jobs;
        metrics.add("pages_decompressed_device", pages_dev);
        metrics.add("pages_decompressed_host", pages_host);
        uint8_t* unc_scratch = nullptr;   // one scratch block for every device-decompressed page of the batch
        if (unc_total > 0) {
            p.unc_device = t.ctx.device;
            p.unc_dev = dev_stage_pool().get((size_t)unc_total + 256, p.unc_device, &p.unc_cap);
            unc_scratch = (uint8_t*)p.unc_dev;
        }
        decomp_jobs.resize(n_jobs);
        parallel_for(p.cols.size(), (unsigned)p.cols.size(), [&](size_t c) {   // (value-initialisation = page faults: one thread per column)
            p.cols[c].pages.resize(npages[c]);
            p.cols[c].dicts.resize(ndicts[c]);
            p.cols[c].secs.resize(nsecs[c]);
        });
        // Phase B (worker pool): pointer fix-ups and the copy of every chunk's descriptors into its slot, rebased
        parallel_for(p.tasks.size(), host_threads, [&](size_t ti) {
            ChunkTask& ct = p.tasks[ti];
            ColState& cs = p.cols[ct.col];
            ChunkPages& cp = ct.out;
            const Slot& sl = slots[ti];
            if (!cp.unc.empty() || cp.gpu_unc_bytes > 0) {
                const uint8_t* dev_base = nullptr;
                if (cp.gpu_unc_bytes > 0) {   // decompressed by pq_decompress below, straight from the chunk bytes in HBM
                    uint8_t* cbase = unc_scratch + sl.unc_off;
                    dev_base = cbase;
                    for (auto& pg : cp.pages)
                        if (pg.job >= 0) pg.job += (int32_t)sl.job_base;
                    for (size_t j = 0; j < cp.jobs.size(); j++) {
                        PqDecompJob jb = cp.jobs[j];
                        jb.dst = cbase + (intptr_t)jb.dst;
                        decomp_jobs[sl.job_base + j] = jb;
                    }
                }
                const uint8_t* host_base = P<uint8_t>(sl.host_unc);
                for (auto& fx : cp.fixes) {
                    const uint8_t* base = fx.dev ? dev_base : host_base;
                    if (fx.page == SIZE_MAX) {
                        cp.dicts[fx.dict].data = base + fx.off;
                        if (fx.sec != SIZE_MAX) cp.secs[fx.sec].ptr = base + fx.off;
                    } else {
                        PqPage& pg = cp.pages[fx.page];
                        pg.def_ptr = pg.def_len ? base + fx.off + (intptr_t)pg.def_ptr : nullptr;
                        intptr_t vo = (intptr_t)pg.val_ptr;
                        pg.val_ptr = base + fx.off + vo;
                        if (fx.sec != SIZE_MAX) cp.secs[fx.sec].ptr = pg.val_ptr;
                    }
                }
            }
            for (size_t i = 0; i < cp.dicts.size(); i++) {
                PqDict d = cp.dicts[i];
                d.value_base += sl.vbase;
                cs.dicts[sl.dict_base + i] = d;
            }
            for (size_t i = 0; i < cp.secs.size(); i++) {
                PqByteSection sc = cp.secs[i];
                sc.value_base += sl.vbase;
                cs.secs[sl.sec_base + i] = sc;
            }
            PqPage* dst = cs.pages.data() + sl.page_base;
            for (size_t i = 0; i < cp.pages.size(); i++) {
                PqPage pg = cp.pages[i];
                if (pg.dict_id >= 0) pg.dict_id += (int32_t)sl.dict_base;
                if (pg.delta_dst16) pg.delta_dst16 += (int32_t)(sl.unc_off / 16);
                pg.plain_value_base += sl.vbase;
                if (cs.shape == pq::SHAPE_LIST) pg.row_start += (int32_t)sl.val_base;
                dst[i] = pg;
            }
        });
        delete tmerge;
        PqDecompOut dec = pq_decompress(wc, decomp_jobs, n_snappy_jobs);
        sg.status = dec.status;
        sg.job_codec.resize(decomp_jobs.size());
        for (size_t j = 0; j < decomp_jobs.size(); j++)
            sg.job_codec[j] = decomp_jobs[j].kind == PQ_JOB_ZSTD ? pq::CODEC_ZSTD : decomp_jobs[j].kind == PQ_JOB_LZ4 ? pq::CODEC_LZ4_RAW : pq::CODEC_SNAPPY;
        bool any_delta = false;
        for (auto& cs : p.cols) any_delta = any_delta || cs.has_delta;
        sg.has_jobs = !decomp_jobs.empty() || any_delta;
        unc_scratch_ptr = unc_scratch;
        status_ptr = P<int32_t>(dec.status);
        decomp_results_buf = dec.results;
        decomp_results = P<PqDecompResult>(dec.results);
        sg.ready = std::move(ready);
        return sg;
    }
    Buf decomp_results_buf;   // keeps the results of the batch being decoded alive
    void check_decomp_status(Task& t, const Staged& sg) {   // synchronises
        if (!sg.has_jobs) return;
        int32_t st = 0;
        to_host(t.ctx, &st, sg.status->ptr, 4);
        if (st != 0) fail(decomp_error(sg, st));
    }
    static std::string decomp_error(const Staged& sg, int32_t st) {
        if (st >= 0x40000000) return "corrupt DELTA_BINARY_PACKED page in the parquet file";
        const size_t j = (size_t)(st - 1);
        const int codec = j < sg.job_codec.size() ? sg.job_codec[j] : pq::CODEC_SNAPPY;
        const char* name = codec == pq::CODEC_ZSTD ? "ZSTD" : codec == pq::CODEC_LZ4_RAW ? "LZ4_RAW" : "Snappy";
        return std::string("corrupt ") + name + " page in the parquet file (decompression job " + std::to_string(j) + ")";
    }

    BatchPtr next(Task& t) override {
        OpTimer timer(metrics, "elapsed_ns");
        retire_fused(t);
        Staged sg = stage_next(t, t.ctx);
        if (!sg.ready) return nullptr;
        return decode_staged(t, sg);
    }
    // the regular path: Arrow columns of the staged batch
    BatchPtr decode_staged(Task& t, Staged& sg) {
        Prepared& p = *sg.ready;
        struct Releaser {
            ParquetScanExec* op;
            Prepared* p;
            cudaStream_t st;
            int exc;
            ~Releaser() {
                if (std::uncaught_exceptions() > exc) {   // decode kernels may still read the landing buffer
                    for (auto& l : op->lanes) cudaStreamSynchronize(l->stream);
                    cudaStreamSynchronize(st);
                }
                op->release(*p);
                op->decomp_results = nullptr;
                op->decomp_results_buf.reset();
            }
        } releaser{this, sg.ready.get(), t.ctx.stream, std::uncaught_exceptions()};
        BatchPtr b;
        {
            OpTimer timer2(metrics, "decode_ns");
            b = build_batch(t, p.cols, p.rows, p.file_segs);   // ends with a stream sync of the task stream, which has joined every lane
            check_decomp_status(t, sg);
        }
        if (p.copy_begin && p.copied) {
            float ms = 0;
            CUDA_OK(cudaEventSynchronize(p.copied));
            CUDA_OK(cudaEventElapsedTime(&ms, p.copy_begin, p.copied));
            metrics.add("h2d_device_us", (int64_t)(ms * 1000));
        }
        metrics.add("output_rows", b->num_rows);
        return b;
    }

    // ------------------------------------------------------------------------------------------ fused scan -> filter -> aggregate
    // (FusedScanSource, operators.h; kernels in k_fused.cu).  A batch whose columns the fused kernels cannot take (strings,
    // INT64 / FLBA physical types, missing statistics of the key, a key range too wide for the direct table) comes back as a
    // regular batch and the caller runs the unfused operators on it.
    struct Inflight {   // a batch whose kernels are still running: its landing buffers are recycled once they are done
        Staged sg;
        cudaEvent_t done = nullptr;
    };
    // Several batches are in flight at a time, on alternating lanes (stream pairs): scout / decompress / fused kernel of one batch
    // are each latency-bound on their own, so the next batches' early stages fill the SMs the current one leaves idle, and the
    // host-side preparation of a batch overlaps the kernels of the previous ones.  The host never waits for a batch unless
    // kMaxInflight of them are queued (their landing buffers are recycled as their completion events fire).
    static constexpr int kFusedLanes = 3, kMaxInflight = 6;
    std::deque<std::unique_ptr<Inflight>> inflight;
    int64_t fused_seq = 0;
    void retire_one(Task& t, bool wait) {
        if (inflight.empty()) return;
        if (!wait && cudaEventQuery(inflight.front()->done) != cudaSuccess) return;
        std::unique_ptr<Inflight> f = std::move(inflight.front());
        inflight.pop_front();
        cudaEventSynchronize(f->done);
        cudaEventDestroy(f->done);
        struct R {
            ParquetScanExec* op;
            Prepared* p;
            ~R() { op->release(*p); }
        } r{this, f->sg.ready.get()};
        if (f->sg.has_jobs) {
            int32_t st = 0;
            CUDA_OK(cudaMemcpy(&st, f->sg.status->ptr, 4, cudaMemcpyDeviceToHost));   // the batch is complete: plain copy, no stream involved
            if (st != 0) fail(decomp_error(f->sg, st));
        }
    }
    void retire_fused(Task& t) {
        while (!inflight.empty()) retire_one(t, true);
        fold_lanes(t);
    }
    void restart(Task& t) override {
        retire_fused(t);
        stop();
        cur.reset();
        file_pos = 0;
        rg_pos = 0;
        producer_started = producer_done = stop_producer = false;
        producer_err.clear();
        for (auto& kv : metrics.values)
            if (kv.first == "output_rows" || kv.first == "fused_batches") kv.second = 0;
        metrics.add("restarted_unfused", 1);
    }
    static bool fused_type_ok(const DType& t) { return t.id == T_INT32 || t.id == T_DATE32 || t.id == T_INT64; }
    bool can_fuse(const FusedAggSpec& spec) const override {
        if (getenv("AURON_DISABLE_FUSED_SCAN_AGG")) return false;
        auto col_ok = [&](int c) { return c >= 0 && c < (int)projection.size() && !is_part_col(projection[c]) && fused_type_ok(table_schema.fields[projection[c]].type); };
        if (!col_ok(spec.key_col)) return false;
        // One predicate COLUMN (any number of conjuncts on it: they fold into one interval).  The kernels loop over predicate columns, but
        // that loop has no GPU parity test yet; until it has one, conjunctions over several columns run operator by operator.
        if (spec.pred_cols.size() > 1) return false;
        for (int c : spec.pred_cols)
            if (!col_ok(c)) return false;
        for (auto& a : spec.accs)
            if (a.col >= 0 && !col_ok(a.col)) return false;
        return (int)spec.accs.size() <= FZ_MAX_ACCS;
    }
    int next_fused(Task& t, const FusedAggSpec& spec, FusedAggState& st, BatchPtr* fallback) override {
        OpTimer timer(metrics, "elapsed_ns");
        const bool multi = !getenv("AURON_FUSED_ONE_LANE");
        const int li = multi ? (int)(fused_seq % kFusedLanes) : 0;
        // lane li = a high-priority stream for the batch's preparation (page decompression, scout: one warp per page, a few
        // long serial chains that leave the SMs mostly idle) + a normal-priority stream for its fused kernel.  While the fused
        // kernel of batch k fills the machine, the preparation of batch k+1 gets the SM slots it needs as soon as it asks.
        if (multi && (int)lanes.size() < 2 * kFusedLanes) {
            for (int i = 0; i < kFusedLanes; i++) lane(t, i, -1);
            for (int i = 0; i < kFusedLanes; i++) lane(t, kFusedLanes + i, 0);
        }
        Ctx& wc = multi ? lane(t, li) : t.ctx;
        Ctx& fc = multi ? lane(t, kFusedLanes + li) : t.ctx;
        {
            OpTimer tr(metrics, "fused_retire_ns");
            while (!inflight.empty() && cudaEventQuery(inflight.front()->done) == cudaSuccess) retire_one(t, false);
            while ((int)inflight.size() >= (multi ? kMaxInflight : 1)) retire_one(t, true);
        }
        Staged sg;
        {
            OpTimer ts(metrics, "fused_stage_ns");
            sg = stage_next(t, wc);
        }
        if (!sg.ready) {
            retire_fused(t);
            return FUSED_END;
        }
        bool ok = false;
        try {
            OpTimer tq(metrics, "fused_enqueue_ns");
            ok = run_fused(t, wc, fc, sg, spec, st);
        } catch (...) {
            cudaStreamSynchronize(wc.stream);
            release(*sg.ready);
            throw;
        }
        if (!ok) {
            retire_fused(t);
            if (&wc != &t.ctx) chain(wc.stream, t.ctx.stream);   // page decompression was queued on the lane
            *fallback = decode_staged(t, sg);
            return FUSED_FALLBACK;
        }
        auto f = std::make_unique<Inflight>();
        CUDA_OK(cudaEventCreateWithFlags(&f->done, cudaEventDisableTiming));
        CUDA_OK(cudaEventRecord(f->done, wc.stream));
        metrics.add("output_rows", sg.ready->rows);
        metrics.add("fused_batches", 1);
        f->sg = std::move(sg);
        inflight.push_back(std::move(f));
        decomp_results = nullptr;
        decomp_results_buf.reset();
        fused_seq++;
        return FUSED_DONE;
    }
    bool run_fused(Task& t, Ctx& wc, Ctx& fc, Staged& sg, const FusedAggSpec& spec, FusedAggState& st) {
        Prepared& p = *sg.ready;
        const int64_t n_rows = p.rows;
        if (n_rows <= 0 || n_rows >= (int64_t)INT32_MAX - FZ_TILE) return false;
        // distinct physical columns
        std::vector<int> used;
        auto phys_of = [&](int c) {
            for (size_t i = 0; i < used.size(); i++)
                if (used[i] == c) return (int)i;
            used.push_back(c);
            return (int)used.size() - 1;
        };
        for (int c : spec.pred_cols) phys_of(c);
        phys_of(spec.key_col);
        for (auto& a : spec.accs)
            if (a.col >= 0) phys_of(a.col);
        for (int c : used) {
            const ColState& cs = p.cols[(size_t)c];
            const DType& ft = proj_field(projection[(size_t)c]).type;
            // (the fused kernels read INT32 values as signed integers: copies and sign extensions only)
            if (cs.leaf < 0 || cs.is_string || cs.el.type != pq::PT_INT32 || !fused_type_ok(ft) || (cs.cv.kind != PQ_CV_COPY && cs.cv.kind != PQ_CV_SEXT)) return false;
        }
        // key range of this batch from the column-chunk statistics; the table is widened to the union
        const ColState& kcs = p.cols[(size_t)spec.key_col];
        if (!kcs.stat_ok) return false;
        long long bmin = kcs.stat_min, bmax = kcs.stat_max;   // min > max: every key of the batch is NULL
        long long umin = bmin, umax = bmax;
        if (st.table && st.has_range) {
            if (bmin <= bmax) {
                umin = std::min<long long>(bmin, st.kmin);
                umax = std::max<long long>(bmax, st.kmax);
            } else {
                umin = st.kmin;
                umax = st.kmax;
            }
        }
        if (umin <= umax && (unsigned long long)umax - (unsigned long long)umin >= (unsigned long long)direct_agg_span_limit()) return false;
        int64_t dict_slots = 0;
        for (auto& d : kcs.dicts) dict_slots += d.num_values;
        if (dict_slots >= (int64_t)1 << 31) return false;

        const int n_tiles = (int)((n_rows + FZ_TILE - 1) / FZ_TILE);
        struct Phys {
            ColDescriptors descr;
            Buf seg_base, segs, first_seg, valid;
        };
        std::vector<Phys> ph(used.size());
        std::vector<FzScoutCol> scout;
        auto tphase = std::make_unique<OpTimer>(metrics, "fused_host_descr_ns");   // host phases of the enqueue, one after the other
        for (size_t u = 0; u < used.size(); u++) {
            ColState& cs = p.cols[(size_t)used[u]];
            const int max_def = cs.el.repetition == 1 ? 1 : 0;
            Phys& x = ph[u];
            x.descr = upload_descriptors(wc, cs);
            std::vector<int32_t> sb(cs.pages.size() + 1, 0);
            for (size_t i = 0; i < cs.pages.size(); i++) {
                const int64_t r0 = cs.pages[i].row_start, n = cs.pages[i].num_values;
                sb[i + 1] = sb[i] + (n > 0 ? (int32_t)((r0 + n - 1) / FZ_TILE - r0 / FZ_TILE + 1) : 0);
            }
            x.seg_base = to_device(wc, sb.data(), sb.size() * 4);
            x.segs = dalloc(wc, (size_t)std::max<int32_t>(sb.back(), 1) * sizeof(FzSeg));
            x.first_seg = dalloc_zero(wc, (size_t)n_tiles * 4);
            if (max_def > 0) x.valid = dalloc_zero(wc, (size_t)n_tiles * (FZ_TILE / 8));
            FzScoutCol sc;
            sc.pages = P<PqPage>(x.descr.pages);
            sc.dicts = P<PqDict>(x.descr.dicts);
            sc.n_pages = (int32_t)cs.pages.size();
            sc.max_def = max_def;
            sc.seg_base = P<int32_t>(x.seg_base);
            sc.segs = P<FzSeg>(x.segs);
            sc.first_seg = P<int32_t>(x.first_seg);
            sc.valid = P<uint32_t>(x.valid);
            scout.push_back(sc);
            if (max_def > 0 && (size_t)used[u] == (size_t)spec.key_col) st.key_nullable = true;
        }
        tphase = std::make_unique<OpTimer>(metrics, "fused_host_scout_ns");
        fz_scout(wc, scout);
        tphase = std::make_unique<OpTimer>(metrics, "fused_host_roles_ns");

        FzLaunch L;
        memset(&L, 0, sizeof(L));
        std::vector<Buf> keep;
        auto add_role = [&](int c, int role) {
            AURON_CHECK(L.ncols < FZ_MAX_COLS, "too many columns in the fused scan");
            const Phys& x = ph[(size_t)phys_of(c)];
            FzColumn& C = L.col[L.ncols];
            C.pages = P<PqPage>(x.descr.pages);
            C.dicts = P<PqDict>(x.descr.dicts);
            C.segs = P<FzSeg>(x.segs);
            C.first_seg = P<int32_t>(x.first_seg);
            C.valid = P<uint32_t>(x.valid);
            C.role = role;
            {   // shared memory for one tile of the column in the TMA-staged kernel: 128 bytes per bit of index width (the writer's
                // width is that of the largest index), run headers, 16-byte alignment at both ends and the window slack; PLAIN pages
                // of a dictionary column are wider than that and stay with the tile kernel
                const ColState& cs = p.cols[(size_t)c];
                int32_t max_dict = 0;
                for (auto& d : cs.dicts) max_dict = std::max(max_dict, d.num_values);
                int bits = 1;
                while (bits < 32 && (1ll << bits) < (int64_t)max_dict) bits++;
                C.stage_cap = cs.dicts.empty() ? 4 * FZ_TILE + 64 : 128 * bits + 80;
                if (cs.el.type != pq::PT_INT32) C.stage_cap = 0;
            }
            return L.ncols++;
        };
        for (size_t i = 0; i < spec.pred_cols.size(); i++) {
            const int c = spec.pred_cols[i];
            const int rc = add_role(c, FZ_PRED);
            const ColState& cs = p.cols[(size_t)c];
            L.col[rc].lo = spec.pred_lo[i];
            L.col[rc].hi = spec.pred_hi[i];
            std::vector<int32_t> off(cs.dicts.size() + 1, 0);
            for (size_t d = 0; d < cs.dicts.size(); d++) off[d + 1] = off[d] + (cs.dicts[d].num_values + 31) / 32;
            Buf doff = to_device(wc, off.data(), off.size() * 4);
            Buf bits = dalloc(wc, (size_t)std::max<int32_t>(off.back(), 1) * 4);
            fz_dict_pass(wc, L.col[rc].dicts, P<int32_t>(doff), (int)cs.dicts.size(), off.back(), spec.pred_lo[i], spec.pred_hi[i], P<uint32_t>(bits));
            L.col[rc].pass_off = P<int32_t>(doff);
            L.col[rc].pass_bits = P<uint32_t>(bits);
            keep.push_back(doff);
            keep.push_back(bits);
        }
        L.npred = L.ncols;
        L.key_col = add_role(spec.key_col, FZ_KEY);
        std::vector<int32_t> dbase(kcs.dicts.size() + 1, 0);
        for (size_t d = 0; d < kcs.dicts.size(); d++) dbase[d + 1] = dbase[d] + kcs.dicts[d].num_values;
        Buf ddbase = to_device(wc, dbase.data(), dbase.size() * 4);
        L.col[L.key_col].dslot_base = P<int32_t>(ddbase);
        std::vector<int> value_role(projection.size(), -1);
        for (auto& a : spec.accs)
            if (a.col >= 0 && a.kind != ACC_COUNT && value_role[(size_t)a.col] < 0) value_role[(size_t)a.col] = add_role(a.col, FZ_VALUE);
        // COUNT(x) only needs x's validity: the key column serves as it is, any other column gets an argument plane
        auto any_role = [&](int c) {
            if (value_role[(size_t)c] >= 0) return value_role[(size_t)c];
            if (c == spec.key_col) return (int)L.key_col;
            return value_role[(size_t)c] = add_role(c, FZ_VALUE);
        };
        // the persistent table
        // The table belongs to the task stream; the lanes only update it.  Creating / widening it is rare (first batch, or a batch
        // whose keys leave the range so far).  No host-side wait: the task stream first waits for everything queued on the lanes
        // (kernels that update the old table), creates / rebases the table, and the lanes wait for that before they go on.
        tphase = std::make_unique<OpTimer>(metrics, "fused_host_table_ns");
        const bool widen = st.table && st.has_range && umin <= umax && (umin < st.kmin || umax > st.kmax);
        if (!st.table || widen || !st.has_range) {
            if (st.table)   // (a table that does not exist yet has no users to wait for)
                for (auto& l : lanes) chain(l->stream, t.ctx.stream);
            if (!st.table) {
                std::vector<AccSpec> specs;
                for (auto& a : spec.accs) {
                    AccSpec s;
                    s.kind = (AccKind)a.kind;
                    s.out_type = a.out_type;
                    s.input_id = a.col;
                    specs.push_back(s);
                }
                st.table = direct_agg_create(t.ctx, specs, umin, umax);
                st.selected = dalloc_zero(t.ctx, 16);   // [0] rows that passed the predicates, [1] tiles done by the TMA-staged kernel
            } else {
                direct_agg_grow(t.ctx, *st.table, umin, umax);
            }
            for (auto& l : lanes) chain(t.ctx.stream, l->stream);
        }
        if (umin <= umax) {
            st.has_range = true;
            st.kmin = umin;
            st.kmax = umax;
        }
        const DirectAggView dv = direct_agg_view(*st.table);
        L.nacc = (int)spec.accs.size();
        tphase = std::make_unique<OpTimer>(metrics, "fused_host_launch_ns");
        Buf dseen = dalloc(wc, (size_t)std::max<int64_t>(dict_slots, 1));
        for (int a = 0; a < L.nacc; a++) {
            FzAcc& A = L.acc[a];
            A.kind = spec.accs[(size_t)a].kind;
            A.col = spec.accs[(size_t)a].col >= 0 ? any_role(spec.accs[(size_t)a].col) : -1;
            A.direct = dv.acc[a];
            A.direct_valid = dv.valid[a];
            Buf d = dalloc(wc, (size_t)std::max<int64_t>(dict_slots, 1) * 8);
            keep.push_back(d);
            A.dspace = P<unsigned long long>(d);
            if (A.direct_valid) {
                Buf v = dalloc(wc, (size_t)std::max<int64_t>(dict_slots, 1));
                keep.push_back(v);
                A.dspace_valid = P<uint8_t>(v);
            }
        }
        L.n_rows = n_rows;
        L.n_tiles = n_tiles;
        L.kmin = dv.kmin;
        L.range = dv.range;
        L.seen_direct = dv.seen;
        L.seen_dspace = P<uint8_t>(dseen);
        L.oor = dv.oor;
        L.selected_rows = P<unsigned long long>(st.selected);
        // SUM(x), COUNT(x) (AVG's partial state) of a narrow x: one atomic per row instead of two.  The SUM word of a dictionary entry
        // holds (count << shift) | sum(x - min) for the batch: sum(x - min) < rows * 2^bits needs bits + ceil(log2 rows) bits, the
        // count the rest.  min / max come from the chunk statistics; a value outside them raises `oor` like a key would.
        if (L.nacc == 2 && L.acc[0].kind == ACC_SUM_I64 && L.acc[1].kind == ACC_COUNT && L.acc[0].col >= 0 && L.acc[0].col == L.acc[1].col &&
            L.acc[0].col != L.key_col && !L.acc[0].direct_valid && !L.acc[1].direct_valid) {
            const ColState& vcs = p.cols[(size_t)spec.accs[0].col];
            if (vcs.stat_ok && vcs.stat_min <= vcs.stat_max) {
                int bits = 1, rbits = 1;
                while (bits < 40 && (vcs.stat_max - vcs.stat_min) >= (1ll << bits)) bits++;
                while ((1ll << rbits) <= n_rows) rbits++;
                if (bits + 2 * rbits + 1 <= 64) {
                    L.pack_bits = bits;
                    L.pack_shift = bits + rbits;
                    L.pack_bias = vcs.stat_min;
                }
            }
        }
        fz_init_dspace(wc, L, dict_slots);
        if (&fc != &wc) chain(wc.stream, fc.stream);
        fz_run(fc, L);
        FzMerge M;
        memset(&M, 0, sizeof(M));
        M.dicts = L.col[L.key_col].dicts;
        M.dslot_base = P<int32_t>(ddbase);
        M.n_dicts = (int32_t)kcs.dicts.size();
        M.nacc = L.nacc;
        for (int a = 0; a < L.nacc; a++) M.acc[a] = L.acc[a];
        M.kmin = dv.kmin;
        M.range = dv.range;
        M.seen_direct = dv.seen;
        M.seen_dspace = P<uint8_t>(dseen);
        M.oor = dv.oor;
        M.pack_shift = L.pack_shift;
        M.pack_bits = L.pack_bits;
        M.pack_bias = L.pack_bias;
        fz_merge(fc, M, dict_slots);
        if (&fc != &wc) chain(fc.stream, wc.stream);   // the batch's buffers are freed (stream-ordered) on wc: after its kernels
        st.rows += n_rows;
        st.batches++;
        return true;
    }
};

OperatorPtr make_parquet_scan(Task& t, const uint8_t* node, size_t n) {
    auto op = std::make_unique<ParquetScanExec>();
    op->name = "ParquetExec";
    op->host_threads = std::max(1u, std::min(32u, usable_cpus()));
    if (const char* e = getenv("AURON_SCAN_THREADS")) op->host_threads = (unsigned)std::max(1, atoi(e));
    if (const char* e = getenv("AURON_SCAN_PREFETCH_DEPTH")) op->prefetch_depth = atoi(e);
    PbReader r(node, n);
    uint32_t f, w;
    std::vector<std::vector<uint8_t>> prune_exprs;
    while (r.next(&f, &w)) {
        if (f == 1 && w == 2) {   // FileScanExecConf
            const uint8_t* cb;
            size_t cn;
            r.bytes_view(&cb, &cn);
            PbReader c(cb, cn);
            uint32_t cf, cw;
            while (c.next(&cf, &cw)) {
                if (cf == 3 && cw == 2) {   // FileGroup{files=1}
                    const uint8_t* gb;
                    size_t gn;
                    c.bytes_view(&gb, &gn);
                    PbReader g(gb, gn);
                    uint32_t gf, gw;
                    while (g.next(&gf, &gw)) {
                        if (gf == 1 && gw == 2) {   // PartitionedFile{path=1,size=2,range=5{start=1,end=2}}
                            const uint8_t* fb;
                            size_t fn;
                            g.bytes_view(&fb, &fn);
                            PbReader pf(fb, fn);
                            uint32_t pff, pfw;
                            PqFileSpec spec;
                            while (pf.next(&pff, &pfw)) {
                                if (pff == 1 && pfw == 2) spec.path = pf.bytes();
                                else if (pff == 2 && pfw == 0) spec.size = (int64_t)pf.varint();
                                else if (pff == 4 && pfw == 2) {   // repeated ScalarValue partition_values {ipc_bytes = 1}
                                    const uint8_t* vb;
                                    size_t vn;
                                    pf.bytes_view(&vb, &vn);
                                    PbReader sv(vb, vn);
                                    uint32_t svf, svw;
                                    Literal lit;
                                    while (sv.next(&svf, &svw)) {
                                        if (svf == 1 && svw == 2) {
                                            const uint8_t* ib;
                                            size_t in;
                                            sv.bytes_view(&ib, &in);
                                            lit = decode_scalar_ipc(ib, in);
                                        } else sv.skip(svw);
                                    }
                                    spec.partition_values.push_back(lit);
                                }
                                else if (pff == 5 && pfw == 2) {
                                    const uint8_t* rb;
                                    size_t rn;
                                    pf.bytes_view(&rb, &rn);
                                    PbReader rr(rb, rn);
                                    uint32_t rf, rw;
                                    spec.range_start = 0;
                                    spec.range_end = 0;
                                    while (rr.next(&rf, &rw)) {
                                        if (rf == 1 && rw == 0) spec.range_start = (int64_t)rr.varint();
                                        else if (rf == 2 && rw == 0) spec.range_end = (int64_t)rr.varint();
                                        else rr.skip(rw);
                                    }
                                } else pf.skip(pfw);
                            }
                            op->files.push_back(spec);
                        } else g.skip(gw);
                    }
                } else if (cf == 4 && cw == 2) {
                    const uint8_t* sb;
                    size_t sn;
                    c.bytes_view(&sb, &sn);
                    op->table_schema = decode_schema(sb, sn);
                } else if (cf == 6 && cw == 0) op->projection.push_back((int)c.varint());
                else if (cf == 6 && cw == 2) {   // packed
                    const uint8_t* pb;
                    size_t pn;
                    c.bytes_view(&pb, &pn);
                    PbReader p(pb, pn);
                    while (!p.done()) op->projection.push_back((int)p.varint());
                } else if (cf == 9 && cw == 2) {
                    const uint8_t* sb;
                    size_t sn;
                    c.bytes_view(&sb, &sn);
                    op->part_schema = decode_schema(sb, sn);
                } else c.skip(cw);
            }
        } else if (f == 3 && w == 2) op->fs_id = r.bytes();
        else if (f == 2 && w == 2) {   // repeated PhysicalExprNode pruning_predicates
            const uint8_t* eb;
            size_t en;
            r.bytes_view(&eb, &en);
            prune_exprs.emplace_back(eb, eb + en);
        } else r.skip(w);
    }
    // row-group pruning is an optimisation: a predicate this engine cannot fold into per-column intervals prunes nothing
    if (!prune_exprs.empty()) {
        try {
            std::vector<ExprPtr> es;
            for (auto& b : prune_exprs) es.push_back(decode_expr(b.data(), b.size()));
            VmProgram pp = compile_predicate(es, op->table_schema);
            if (!predicate_intervals(pp, &op->prune_cols, &op->prune_lo, &op->prune_hi)) op->prune_cols.clear();
        } catch (const std::exception&) {
            op->prune_cols.clear();
        }
    }
    if (op->projection.empty())
        for (size_t i = 0; i < op->table_schema.fields.size() + op->part_schema.fields.size(); i++) op->projection.push_back((int)i);
    for (int p : op->projection) {
        AURON_CHECK(p >= 0 && p < (int)(op->table_schema.fields.size() + op->part_schema.fields.size()), "scan projection out of range");
        op->out_schema.fields.push_back(op->proj_field(p));
        const Field& f = op->proj_field(p);
        if (f.type.id == T_LIST && op->is_part_col(p)) fail("ParquetScanExec: list column " + f.name + " (" + f.type.str() + ") is not supported as a partition column");
    }
    (void)t;
    return op;
}

}  // namespace auron
