// shuffle_writer.cc -- ShuffleWriterExec (rows S2, S4-S6 of SURVEY.md section 8a).  Mirrors
// ShuffleWriterExec::execute (datafusion-ext-plans/src/shuffle_writer_exec.rs:106-168), the repartitioners
// (shuffle/sort_repartitioner.rs:123-254, single_repartitioner.rs:64-97), BufferedData::write
// (shuffle/buffered_data.rs:123-158) and IpcCompressionWriter (datafusion-ext-commons/src/io/ipc_compression.rs:35-113).
//
// Per device chunk: partition ids on device (k_hash.cu), stable counting sort of row ids (k_sort.cu), one gather
// into a partition-contiguous batch, byte-plane serialisation of all partitions in one pass (k_serde.cu), one
// D2H, then LZ4-frame / ZSTD block compression per partition on the host cores (system liblz4 / libzstd via
// dlopen; the reference uses lz4_flex frame / zstd, ipc_compression.rs:178-197).  Output files:
//   data  = for each partition, its blocks from every chunk, concatenated     (sort_repartitioner.rs:217-249)
//   block = u32_le compressed_len | codec stream                              (ipc_compression.rs:84-103)
//   index = (N+1) little-endian i64 offsets, first = 0                        (sort_repartitioner.rs:166-193)
#include <dlfcn.h>

#include <atomic>
#include <cstdio>
#include <mutex>
#include <thread>

#include <fcntl.h>
#include <sys/mman.h>
#include <unistd.h>

#include "exchange.h"
#include "host_pool.h"
#include "../../include/auron_b200.h"
#include "operators.h"
#include "pb.h"

namespace auron {

namespace {
typedef size_t (*lz4f_bound_fn)(size_t, const void*);
typedef size_t (*lz4f_compress_fn)(void*, size_t, const void*, size_t, const void*);
typedef unsigned (*lz4f_iserror_fn)(size_t);
typedef size_t (*zstd_bound_fn)(size_t);
typedef size_t (*zstd_compress_fn)(void*, size_t, const void*, size_t, int);
typedef unsigned (*zstd_iserror_fn)(size_t);

struct Codecs {
    lz4f_bound_fn lz4_bound = nullptr;
    lz4f_compress_fn lz4_compress = nullptr;
    lz4f_iserror_fn lz4_iserr = nullptr;
    zstd_bound_fn z_bound = nullptr;
    zstd_compress_fn z_compress = nullptr;
    zstd_iserror_fn z_iserr = nullptr;
    Codecs() {
        if (void* h = dlopen("liblz4.so.1", RTLD_NOW)) {
            lz4_bound = (lz4f_bound_fn)dlsym(h, "LZ4F_compressFrameBound");
            lz4_compress = (lz4f_compress_fn)dlsym(h, "LZ4F_compressFrame");
            lz4_iserr = (lz4f_iserror_fn)dlsym(h, "LZ4F_isError");
        }
        if (void* h = dlopen("libzstd.so.1", RTLD_NOW)) {
            z_bound = (zstd_bound_fn)dlsym(h, "ZSTD_compressBound");
            z_compress = (zstd_compress_fn)dlsym(h, "ZSTD_compress");
            z_iserr = (zstd_iserror_fn)dlsym(h, "ZSTD_isError");
        }
    }
};
const Codecs& codecs() {
    static Codecs c;
    return c;
}

// one block: u32_le compressed_len | codec stream
void compress_block(bool zstd, int zstd_level, const uint8_t* in, size_t n, std::vector<uint8_t>& out) {
    const Codecs& c = codecs();
    size_t bound, written;
    if (zstd) {
        AURON_CHECK(c.z_compress, "libzstd.so.1 not available");
        bound = c.z_bound(n);
        out.resize(4 + bound);
        written = c.z_compress(out.data() + 4, bound, in, n, zstd_level);   // spark.io.compression.zstd.level (ipc_compression.rs:186-193)
        AURON_CHECK(!c.z_iserr(written), "zstd compression failed");
    } else {
        AURON_CHECK(c.lz4_compress, "liblz4.so.1 not available");
        bound = c.lz4_bound(n, nullptr);
        out.resize(4 + bound);
        written = c.lz4_compress(out.data() + 4, bound, in, n, nullptr);
        AURON_CHECK(!c.lz4_iserr(written), "lz4 frame compression failed");
    }
    uint32_t len = (uint32_t)written;
    memcpy(out.data(), &len, 4);
    out.resize(4 + written);
}
}  // namespace

struct ShuffleWriterExec : Operator {
    int kind = 1;   // 1 single, 2 hash, 3 round robin, 4 range
    std::vector<ExprPtr> hash_exprs;
    // range partitioning: sort expressions + one bound column per expression (num_parts - 1 rows, ascending in sort order)
    std::vector<SortExprSpec> range_keys;
    std::vector<HostArray> range_bounds_host;
    std::vector<ColumnPtr> range_bounds;
    int64_t num_parts = 1;
    std::string data_file, index_file;
    bool done = false;
    bool zstd = false;
    int zstd_level = 1;
    // one finished chunk: the compressed blocks of every partition, back to back, in one host buffer
    struct ChunkOut {
        uint8_t* bytes = nullptr;          // pinned (from pinned_pool) when pinned_cap > 0, else owned
        size_t pinned_cap = 0;
        std::vector<uint8_t> owned;
        std::vector<int64_t> part_off;     // num_parts + 1 offsets into bytes
        int spill = -1;                    // >= 0: the bytes live in spill file `spill` at `spill_off` (bytes == nullptr)
        int64_t spill_off = 0;
    };
    std::vector<ChunkOut> chunks;
    // Memory-bounded buffering (sort_repartitioner.rs:98-112: the repartitioner spills under memory pressure).  Finished chunks wait in
    // pinned host memory for write_files(); once more than `spill_budget` bytes wait (AURON_SHUFFLE_SPILL_BYTES, default 16 GB) they
    // are appended to a spill file next to the data file and their memory goes back to the pool.  write_files() then takes a
    // partition's blocks from memory or from the spill files, in chunk order, so the .data file is byte-identical either way.
    int64_t buffered = 0, spill_budget = -1;
    std::vector<int> spill_fds;
    std::vector<std::string> spill_paths;
    void spill_chunks(Task&) {
        OpTimer timer(metrics, "spill_ns");
        const std::string path = data_file + ".spill" + std::to_string(spill_fds.size());
        int fd = open(path.c_str(), O_RDWR | O_CREAT | O_TRUNC, 0600);
        AURON_CHECK(fd >= 0, "cannot create shuffle spill file " + path);
        spill_fds.push_back(fd);
        spill_paths.push_back(path);
        int64_t off = 0;
        for (auto& c : chunks) {
            if (c.spill >= 0 || !c.bytes) continue;
            const int64_t len = c.part_off.back();
            int64_t done = 0;
            while (done < len) {
                ssize_t w = pwrite(fd, c.bytes + done, (size_t)(len - done), off + done);
                AURON_CHECK(w > 0, "short write on " + path);
                done += w;
            }
            c.spill = (int)spill_fds.size() - 1;
            c.spill_off = off;
            off += len;
            if (c.pinned_cap) pinned_pool().put(c.bytes, c.pinned_cap);
            c.pinned_cap = 0;
            c.owned = std::vector<uint8_t>();
            c.bytes = nullptr;
            metrics.add("mem_spill_count", 1);
            metrics.add("mem_spill_size", len);
        }
        buffered = 0;
    }
    void drop_spills() {
        for (int fd : spill_fds) close(fd);
        for (auto& p : spill_paths) unlink(p.c_str());
        spill_fds.clear();
        spill_paths.clear();
    }
    int64_t rows_so_far = 0;
    bool host_lz4 = getenv("AURON_HOST_LZ4") != nullptr;   // AURON_HOST_LZ4=1: compress LZ4 blocks with liblz4 on the host cores

    std::string describe() const override {
        static const char* kinds[] = {"?", "single", "hash", "round_robin", "range"};
        std::string o = std::string("\"partitioning\":\"") + (kind >= 1 && kind <= 4 ? kinds[kind] : "?") + "\",\"partition_count\":" + std::to_string(num_parts) +
                        ",\"data_file\":" + json_quote(data_file) + ",\"index_file\":" + json_quote(index_file) + ",\"codec\":\"" + (zstd ? "zstd" : "lz4") + "\",\"exprs\":[";
        for (size_t i = 0; i < hash_exprs.size(); i++) o += (i ? "," : "") + json_quote(expr_to_string(*hash_exprs[i]));
        for (size_t i = 0; i < range_keys.size(); i++)
            o += (i ? "," : "") + json_quote(expr_to_string(*range_keys[i].expr) + (range_keys[i].asc ? " ASC" : " DESC") + (range_keys[i].nulls_first ? " NULLS FIRST" : " NULLS LAST"));
        o += "],\"range_bound_rows\":[";
        for (size_t i = 0; i < range_bounds_host.size(); i++) o += (i ? "," : "") + std::to_string(range_bounds_host[i].len);
        return o + "]";
    }
    ~ShuffleWriterExec() override {
        for (auto& c : chunks)
            if (c.pinned_cap) pinned_pool().put(c.bytes, c.pinned_cap);
        drop_spills();
    }

    // LZ4 frames produced on the GPU (k_lz4.cu): compress 64 KB blocks, size them, assemble the partition streams, one D2H
    ChunkOut compress_on_device(Ctx& ctx, const SerializedParts& ser) {
        ChunkOut out;
        out.part_off.assign((size_t)num_parts + 1, 0);
        const uint8_t* raw = P<uint8_t>(ser.bytes);
        std::vector<Lz4Block> blocks;
        std::vector<int32_t> first_block((size_t)num_parts + 1, 0);
        int64_t scratch = 0;
        for (int64_t p = 0; p < num_parts; p++) {
            first_block[(size_t)p] = (int32_t)blocks.size();
            for (int64_t o = ser.part_offsets[p]; o < ser.part_offsets[p + 1]; o += kLz4BlockBytes) {
                int32_t len = (int32_t)std::min<int64_t>(kLz4BlockBytes, ser.part_offsets[p + 1] - o);
                blocks.push_back(Lz4Block{raw + o, (uint8_t*)(intptr_t)scratch, len, 0});
                scratch += (lz4_block_bound(len) + 15) & ~(int64_t)15;
            }
        }
        first_block[(size_t)num_parts] = (int32_t)blocks.size();
        const int nb = (int)blocks.size();
        if (nb == 0) return out;
        Buf dscratch = dalloc(ctx, (size_t)scratch);
        for (auto& b : blocks) b.dst = P<uint8_t>(dscratch) + (intptr_t)b.dst;
        Buf dblocks = to_device(ctx, blocks.data(), blocks.size() * sizeof(Lz4Block));
        Buf dsizes = dalloc(ctx, (size_t)nb * 4);
        lz4_compress_blocks(ctx, P<Lz4Block>(dblocks), nb, P<int32_t>(dsizes));
        std::vector<int32_t> sizes((size_t)nb);
        to_host(ctx, sizes.data(), dsizes->ptr, (size_t)nb * 4);
        // layout: per non-empty partition  u32 frame_len | frame header (7) | { u32 size | data }* | u32 end mark
        static const uint8_t kHeader[7] = {0x04, 0x22, 0x4D, 0x18, 0x60, 0x40, 0x82};   // magic, FLG (v1, independent blocks), BD (64 KB), HC
        std::vector<Lz4Place> places((size_t)nb);
        int64_t pos = 0;
        for (int64_t p = 0; p < num_parts; p++) {
            out.part_off[(size_t)p] = pos;
            const int b0 = first_block[(size_t)p], b1 = first_block[(size_t)p + 1];
            if (b0 == b1) continue;
            int64_t frame = 7 + 4;
            for (int b = b0; b < b1; b++) frame += 4 + std::min(sizes[(size_t)b], blocks[(size_t)b].len);
            AURON_CHECK(frame < (int64_t)UINT32_MAX, "shuffle block too large");
            int64_t w = pos + 4 + 7;
            for (int b = b0; b < b1; b++) {
                const bool stored = sizes[(size_t)b] >= blocks[(size_t)b].len;
                Lz4Place& pl = places[(size_t)b];
                memset(&pl, 0, sizeof(pl));
                pl.src = stored ? blocks[(size_t)b].src : blocks[(size_t)b].dst;
                pl.len = stored ? blocks[(size_t)b].len : sizes[(size_t)b];
                pl.size_word = (uint32_t)pl.len | (stored ? 0x80000000u : 0u);
                pl.dst = (uint8_t*)(intptr_t)w;
                pl.flags = (b == b0 ? 1u : 0u) | (b == b1 - 1 ? 2u : 0u);
                pl.stream_len = (uint32_t)frame;
                memcpy(pl.header, kHeader, 7);
                w += 4 + pl.len;
            }
            pos += 4 + frame;
        }
        out.part_off[(size_t)num_parts] = pos;
        Buf image = dalloc(ctx, (size_t)pos + 16);
        for (auto& pl : places) pl.dst = P<uint8_t>(image) + (intptr_t)pl.dst;
        Buf dplaces = to_device(ctx, places.data(), places.size() * sizeof(Lz4Place));
        lz4_assemble(ctx, P<Lz4Place>(dplaces), nb);
        out.bytes = (uint8_t*)pinned_pool().get((size_t)pos + 64, &out.pinned_cap);
        to_host(ctx, out.bytes, image->ptr, (size_t)pos);
        return out;
    }

    // ZSTD (and AURON_HOST_LZ4=1): raw partition bytes to pinned host memory, one block per partition on the worker pool
    ChunkOut compress_on_host(Ctx& ctx, const SerializedParts& ser) {
        ChunkOut out;
        out.part_off.assign((size_t)num_parts + 1, 0);
        const int64_t total = ser.part_offsets.back();
        size_t cap = 0;
        uint8_t* host = (uint8_t*)pinned_pool().get((size_t)total + 64, &cap);
        std::vector<std::vector<uint8_t>> blocks((size_t)num_parts);
        try {
            to_host(ctx, host, ser.bytes->ptr, (size_t)total);
            parallel_for((size_t)num_parts, 32, [&](size_t p) {
                int64_t b = ser.part_offsets[p], e = ser.part_offsets[p + 1];
                if (e > b) compress_block(zstd, zstd_level, host + b, (size_t)(e - b), blocks[p]);
            });
        } catch (...) {
            pinned_pool().put(host, cap);
            throw;
        }
        pinned_pool().put(host, cap);
        int64_t pos = 0;
        for (int64_t p = 0; p < num_parts; p++) {
            out.part_off[(size_t)p] = pos;
            pos += (int64_t)blocks[(size_t)p].size();
        }
        out.part_off[(size_t)num_parts] = pos;
        out.owned.resize((size_t)pos);
        parallel_for((size_t)num_parts, 16, [&](size_t p) {
            if (!blocks[p].empty()) memcpy(out.owned.data() + out.part_off[p], blocks[p].data(), blocks[p].size());
        });
        out.bytes = out.owned.data();
        return out;
    }

    // evaluate_range_partition_ids + get_partition (shuffle/mod.rs:204-262): partition = number of bound rows that sort strictly
    // before the key row.  On the device: sort [key rows ++ bound rows] once with the stable key sort (bounds last, so a bound
    // equal to a key stays behind it), then the partition of a key row is the number of bound rows in front of it.
    Buf range_partition_ids(Task& t, const Batch& in) {
        Ctx& ctx = t.ctx;
        const int64_t n = in.num_rows;
        if (range_bounds.empty())
            for (auto& h : range_bounds_host) range_bounds.push_back(host_array_to_device(ctx, h));
        AURON_CHECK(range_bounds.size() == range_keys.size(), "range partitioning: one bound list per sort expression expected");
        const int64_t nb = range_bounds.empty() ? 0 : range_bounds[0]->len;
        std::vector<SortKeySpec> specs;
        for (size_t k = 0; k < range_keys.size(); k++) {
            ColumnPtr kc = eval_to_column(t, range_keys[k].expr, children[0]->out_schema, in);
            AURON_CHECK(kc->type == range_bounds[k]->type, "range partitioning: bound type " + range_bounds[k]->type.str() + " != key type " + kc->type.str());
            AURON_CHECK(range_bounds[k]->len == nb, "range partitioning: ragged bound lists");
            specs.push_back({concat_columns(ctx, {kc, range_bounds[k]}), range_keys[k].asc, range_keys[k].nulls_first});
        }
        Buf perm = sort_indices(ctx, specs, n + nb);
        return bound_ranks(ctx, P<int32_t>(perm), n, nb);
    }

    void write_chunk(Task& t, const BatchPtr& in) {
        Ctx& ctx = t.ctx;
        int64_t n = in->num_rows;
        std::vector<int64_t> row_off(num_parts + 1, 0);
        BatchPtr sorted = in;
        if (num_parts > 1) {
            OpTimer timer(metrics, "partition_ns");
            Buf pids;
            if (kind == 2) {
                std::vector<ColumnPtr> keys;
                for (auto& e : hash_exprs) keys.push_back(eval_to_column(t, e, children[0]->out_schema, *in));
                pids = murmur3_partition_ids(ctx, keys, n, (int32_t)num_parts, 42);
            } else if (kind == 3) {
                // sort_batches_by_partition_id (buffered_data.rs:291-312): the first row of a flush starts at
                // (partition_id * 1000193 + rows written so far) % N
                int64_t start = (int64_t)(((uint64_t)t.partition_id * 1000193ull + (uint64_t)rows_so_far) % (uint64_t)num_parts);
                pids = round_robin_partition_ids(ctx, n, start, (int32_t)num_parts);
            } else {
                pids = range_partition_ids(t, *in);
            }
            Buf rows, offs;
            partition_rows(ctx, P<int32_t>(pids), n, (int32_t)num_parts, &rows, &offs);
            to_host(ctx, row_off.data(), offs->ptr, (size_t)(num_parts + 1) * 8);
            sorted = take_batch(ctx, *in, P<int32_t>(rows), n, false);
        } else {
            row_off[1] = n;
        }
        SerializedParts ser;
        {
            OpTimer timer(metrics, "serde_ns");
            ser = serialize_partitions(ctx, *sorted, row_off);
        }
        metrics.add("data_size", ser.part_offsets.back());
        {
            OpTimer timer(metrics, "compress_ns");
            chunks.push_back((zstd || host_lz4) ? compress_on_host(ctx, ser) : compress_on_device(ctx, ser));
        }
        if (!is_ipc_writer && data_file.rfind("nccl", 0) != 0) {
            if (spill_budget < 0) spill_budget = getenv("AURON_SHUFFLE_SPILL_BYTES") ? atoll(getenv("AURON_SHUFFLE_SPILL_BYTES")) : (int64_t)16 << 30;
            buffered += chunks.back().part_off.back();
            if (buffered > spill_budget) spill_chunks(t);
        }
        rows_so_far += n;
    }

    void write_files() {
        OpTimer timer(metrics, "write_ns");
        // .data = for each partition, its blocks of every chunk in chunk order; all positions are known up front, so the
        // segments are written with pwrite from the worker pool
        std::vector<int64_t> offsets((size_t)num_parts + 1, 0);
        struct Seg {
            const uint8_t* src;   // nullptr: read from spill file `fd` at `off`
            int64_t len, pos;
            int fd;
            int64_t off;
        };
        std::vector<Seg> segs;
        int64_t pos = 0;
        for (int64_t p = 0; p < num_parts; p++) {
            offsets[(size_t)p] = pos;
            for (auto& ch : chunks) {
                int64_t b = ch.part_off[(size_t)p], e = ch.part_off[(size_t)p + 1];
                if (e == b) continue;
                segs.push_back(ch.spill >= 0 ? Seg{nullptr, e - b, pos, spill_fds[(size_t)ch.spill], ch.spill_off + b} : Seg{ch.bytes + b, e - b, pos, -1, 0});
                pos += e - b;
            }
        }
        offsets[(size_t)num_parts] = pos;
        int fd = open(data_file.c_str(), O_RDWR | O_CREAT | O_TRUNC, 0644);
        AURON_CHECK(fd >= 0, "cannot create shuffle data file " + data_file);
        if (pos > 0 && ftruncate(fd, pos) != 0) {
            close(fd);
            fail("cannot size shuffle data file " + data_file);
        }
        // Buffered writes to one file serialise on the inode lock; a shared
        // mapping lets the worker pool fault and fill pages in parallel.  pwrite stays as the fallback.
        const unsigned wthreads = getenv("AURON_SHUFFLE_WRITE_THREADS") ? (unsigned)std::max(1, atoi(getenv("AURON_SHUFFLE_WRITE_THREADS"))) : 32u;
        void* map = pos > 0 && !getenv("AURON_SHUFFLE_PWRITE") ? mmap(nullptr, (size_t)pos, PROT_READ | PROT_WRITE, MAP_SHARED, fd, 0) : MAP_FAILED;
        try {
            if (map != MAP_FAILED) {
                struct Piece {
                    const uint8_t* src;
                    int64_t len, pos;
                    int fd;
                    int64_t off;
                };
                std::vector<Piece> pieces;
                const int64_t kPiece = 2 << 20;
                for (auto& sg : segs)
                    for (int64_t o = 0; o < sg.len; o += kPiece) pieces.push_back(Piece{sg.src ? sg.src + o : nullptr, std::min(kPiece, sg.len - o), sg.pos + o, sg.fd, sg.off + o});
                parallel_for(pieces.size(), wthreads, [&](size_t i) {
                    uint8_t* dst = (uint8_t*)map + pieces[i].pos;
#ifdef MADV_POPULATE_WRITE
                    {   // allocate the piece's pages in one call instead of one write fault per page (Linux 5.14+; failure is harmless)
                        const uintptr_t a = (uintptr_t)dst & ~(uintptr_t)4095, e = ((uintptr_t)dst + (size_t)pieces[i].len + 4095) & ~(uintptr_t)4095;
                        (void)madvise((void*)a, (size_t)(e - a), MADV_POPULATE_WRITE);
                    }
#endif
                    if (pieces[i].src) {
                        memcpy(dst, pieces[i].src, (size_t)pieces[i].len);
                    } else {   // spilled: straight from the spill file into the mapping
                        int64_t done = 0;
                        while (done < pieces[i].len) {
                            ssize_t r = pread(pieces[i].fd, dst + done, (size_t)(pieces[i].len - done), pieces[i].off + done);
                            AURON_CHECK(r > 0, "short read on a shuffle spill file");
                            done += r;
                        }
                    }
                });
                munmap(map, (size_t)pos);
            } else {
                parallel_for(segs.size(), wthreads, [&](size_t i) {
                    std::vector<uint8_t> tmp;
                    const uint8_t* src = segs[i].src;
                    if (!src) {   // spilled segment: through a bounce buffer
                        tmp.resize((size_t)segs[i].len);
                        int64_t got = 0;
                        while (got < segs[i].len) {
                            ssize_t r = pread(segs[i].fd, tmp.data() + got, (size_t)(segs[i].len - got), segs[i].off + got);
                            AURON_CHECK(r > 0, "short read on a shuffle spill file");
                            got += r;
                        }
                        src = tmp.data();
                    }
                    int64_t done = 0;
                    while (done < segs[i].len) {
                        ssize_t w = pwrite(fd, src + done, (size_t)(segs[i].len - done), segs[i].pos + done);
                        AURON_CHECK(w > 0, "short write on " + data_file);
                        done += w;
                    }
                });
            }
        } catch (...) {
            if (map != MAP_FAILED) munmap(map, (size_t)pos);
            close(fd);
            throw;
        }
        close(fd);
        drop_spills();
        FILE* xf = fopen(index_file.c_str(), "wb");
        AURON_CHECK(xf, "cannot create shuffle index file " + index_file);
        AURON_CHECK(fwrite(offsets.data(), 8, offsets.size(), xf) == offsets.size(), "short write on " + index_file);
        fclose(xf);
        metrics.add("output_rows", rows_so_far);
    }

    // in-box repartition: output_data_file = "nccl://<name>" turns the writer into an exchange whose output stream is
    // the set of rows this rank owns after the all-to-all (so the next stage can be chained in the same task plan);
    // "nccl-bcast://<name>" is the broadcast exchange (BroadcastExchangeExec on the Spark side: the build side of a broadcast
    // join is collected from every partition and replicated) as an all-gather-v over NVLink
    BatchPtr exchange(Task& t) {
        std::vector<BatchPtr> all;
        while (BatchPtr b = children[0]->next(t)) {
            AURON_CHECK(t.is_running(), "task killed");
            if (b->num_rows) all.push_back(b);
        }
        BatchPtr in;
        if (all.empty()) {
            in = std::make_shared<Batch>();
            for (auto& f : out_schema.fields) in->cols.push_back(make_column(t.ctx, f.type, 0, false));
        } else in = concat_batches(t.ctx, all);
        all.clear();
        int64_t n = in->num_rows;
        if (data_file.rfind("nccl-bcast://", 0) == 0) {   // broadcast exchange: every rank ends up with the rows of all ranks
            int64_t sent = 0;
            BatchPtr out;
            {
                OpTimer timer(metrics, "exchange_ns");
                out = nccl_exchange(t.ctx, *in, {}, 0, &sent);
            }
            metrics.add("data_size", sent);
            metrics.add("output_rows", out->num_rows);
            return out;
        }
        AURON_CHECK(kind == 2, "the NCCL exchange implements hash repartitioning");
        std::vector<ColumnPtr> keys;
        for (auto& e : hash_exprs) keys.push_back(eval_to_column(t, e, children[0]->out_schema, *in));
        Buf pids = murmur3_partition_ids(t.ctx, keys, n, (int32_t)num_parts, 42);
        Buf rows, offs;
        partition_rows(t.ctx, P<int32_t>(pids), n, (int32_t)num_parts, &rows, &offs);
        std::vector<int64_t> row_off(num_parts + 1, 0);
        to_host(t.ctx, row_off.data(), offs->ptr, (size_t)(num_parts + 1) * 8);
        BatchPtr sorted = take_batch(t.ctx, *in, P<int32_t>(rows), n, false);
        int64_t sent = 0;
        BatchPtr out;
        {
            OpTimer timer(metrics, "exchange_ns");
            out = nccl_exchange(t.ctx, *sorted, row_off, num_parts, &sent);
        }
        metrics.add("data_size", sent);
        metrics.add("output_rows", out->num_rows);
        return out;
    }

    // IpcWriterExec (ipc_writer_exec.rs:106-190): the same serialisation + block compression, one partition, every finished chunk of
    // blocks handed to the consumer callback as soon as it exists
    std::string ipc_consumer_id;
    bool is_ipc_writer = false;
    void deliver_chunks(Task& t) {
        AURON_CHECK(t.cb && t.cb->write_ipc, "IpcWriterExec needs the write_ipc callback");
        for (auto& ch : chunks) {
            const int64_t b = ch.part_off[0], e = ch.part_off[1];
            if (e > b && t.cb->write_ipc(t.cb->user, ipc_consumer_id.c_str(), ch.bytes + b, e - b) < 0) fail("write_ipc failed for resource " + ipc_consumer_id);
            metrics.add("data_size_written", e - b);
        }
        chunks.clear();
    }

    BatchPtr next(Task& t) override {
        if (done) return nullptr;
        done = true;
        if (is_ipc_writer) {
            while (BatchPtr b = children[0]->next(t)) {
                AURON_CHECK(t.is_running(), "task killed");
                if (b->num_rows == 0) continue;
                write_chunk(t, b);
                deliver_chunks(t);
            }
            metrics.add("output_rows", rows_so_far);
            return nullptr;
        }
        if (data_file.rfind("nccl://", 0) == 0 || data_file.rfind("nccl-bcast://", 0) == 0) return exchange(t);
        while (BatchPtr b = children[0]->next(t)) {
            AURON_CHECK(t.is_running(), "task killed");
            if (b->num_rows == 0) continue;
            write_chunk(t, b);
        }
        write_files();
        return nullptr;   // the output stream of a shuffle writer is empty (shuffle/mod.rs:61-108)
    }
};

OperatorPtr make_ipc_writer(Task& t, OperatorPtr input, const std::string& consumer_id) {
    auto op = std::make_unique<ShuffleWriterExec>();
    op->name = "IpcWriterExec";
    op->out_schema = input->out_schema;
    op->kind = 1;
    op->num_parts = 1;
    op->is_ipc_writer = true;
    op->ipc_consumer_id = consumer_id;
    op->zstd = t.conf("SPARK_IO_COMPRESSION_CODEC", "AURON_IO_COMPRESSION_CODEC", "lz4") == "zstd";
    op->zstd_level = atoi(t.conf("SPARK_IO_COMPRESSION_ZSTD_LEVEL", "AURON_IO_COMPRESSION_ZSTD_LEVEL", "1").c_str());
    reject_list_exprs(op->hash_exprs, input->out_schema, "a shuffle partitioning key");
    for (auto& k : op->range_keys) reject_list_exprs({k.expr}, input->out_schema, "a shuffle partitioning key");
    op->children.push_back(std::move(input));
    return op;
}

OperatorPtr make_shuffle_writer(Task& t, OperatorPtr input, const uint8_t* node, size_t n) {
    auto op = std::make_unique<ShuffleWriterExec>();
    op->name = "ShuffleWriterExec";
    op->out_schema = input->out_schema;
    PbReader r(node, n);
    uint32_t f, w;
    while (r.next(&f, &w)) {
        if (f == 2 && w == 2) {   // PhysicalRepartition oneof
            const uint8_t* pb;
            size_t pn;
            r.bytes_view(&pb, &pn);
            PbReader p(pb, pn);
            uint32_t pf, pw;
            while (p.next(&pf, &pw)) {
                if (pw != 2) {
                    p.skip(pw);
                    continue;
                }
                const uint8_t* sb;
                size_t sn;
                p.bytes_view(&sb, &sn);
                PbReader s(sb, sn);
                uint32_t sf, sw;
                op->kind = (int)pf;
                AURON_CHECK(pf >= 1 && pf <= 4, "unknown repartition kind");
                while (s.next(&sf, &sw)) {
                    if (pf == 4) {   // PhysicalRangeRepartition{sort_expr = 1 (SortExecNode), partition_count = 2, list_value = 3 (ScalarValue)*}
                        if (sf == 1 && sw == 2) {
                            const uint8_t* nb;
                            size_t nn;
                            s.bytes_view(&nb, &nn);
                            PbReader sn(nb, nn);
                            uint32_t nf, nw;
                            while (sn.next(&nf, &nw)) {
                                if (nf == 2 && nw == 2) {
                                    const uint8_t* eb;
                                    size_t en;
                                    sn.bytes_view(&eb, &en);
                                    op->range_keys.push_back(decode_sort_expr(eb, en));
                                } else sn.skip(nw);
                            }
                        } else if (sf == 2 && sw == 0) op->num_parts = (int64_t)s.varint();
                        else if (sf == 3 && sw == 2) {
                            const uint8_t* vb;
                            size_t vn;
                            s.bytes_view(&vb, &vn);
                            PbReader sv(vb, vn);
                            uint32_t vf, vw;
                            while (sv.next(&vf, &vw)) {
                                if (vf == 1 && vw == 2) {
                                    const uint8_t* ib;
                                    size_t in_;
                                    sv.bytes_view(&ib, &in_);
                                    op->range_bounds_host.push_back(decode_list_scalar_ipc(ib, in_));
                                } else sv.skip(vw);
                            }
                        } else s.skip(sw);
                        continue;
                    }
                    if (pf == 2 && sf == 1 && sw == 2) {
                        const uint8_t* eb;
                        size_t en;
                        s.bytes_view(&eb, &en);
                        ExprPtr he = decode_expr(eb, en);
                        AURON_CHECK(he != nullptr, "hash partitioning: empty expression");
                        op->hash_exprs.push_back(he);
                    } else if (((pf == 2 && sf == 2) || (pf != 2 && sf == 1)) && sw == 0) op->num_parts = (int64_t)s.varint();
                    else s.skip(sw);
                }
            }
        } else if (f == 3 && w == 2) op->data_file = r.bytes();
        else if (f == 4 && w == 2) op->index_file = r.bytes();
        else r.skip(w);
    }
    AURON_CHECK(op->num_parts >= 1 && op->num_parts < (1 << 24), "shuffle writer: partition count out of range (1 .. 2^24 - 1)");
    if (op->kind == 1) op->num_parts = 1;   // SingleShuffleRepartitioner (single_repartitioner.rs:64-97)
    if (op->kind == 4 && op->num_parts == 1) op->kind = 1;   // planner.rs:1161-1162
    if (op->kind == 4)
        for (auto& h : op->range_bounds_host) AURON_CHECK(h.len == op->num_parts - 1, "range partitioning needs partition_count - 1 bounds");
    // spark.io.compression.codec (lz4 | zstd) and spark.io.compression.zstd.level (conf.rs:46-47, ipc_compression.rs:180-200)
    op->zstd = t.conf("SPARK_IO_COMPRESSION_CODEC", "AURON_IO_COMPRESSION_CODEC", "lz4") == "zstd";
    op->zstd_level = atoi(t.conf("SPARK_IO_COMPRESSION_ZSTD_LEVEL", "AURON_IO_COMPRESSION_ZSTD_LEVEL", "1").c_str());
    reject_list_exprs(op->hash_exprs, input->out_schema, "a shuffle partitioning key");
    for (auto& k : op->range_keys) reject_list_exprs({k.expr}, input->out_schema, "a shuffle partitioning key");
    op->children.push_back(std::move(input));
    return op;
}

}  // namespace auron
